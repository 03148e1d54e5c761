"""The MM_LLMs forward pass expressed over the sm_90a kernel library (ops.py -> libmacaw_b200.so).

Every arithmetic step of the reference hot path (reference: /root/reference/modeling.py:941-1118 and the torch /
transformers modules it delegates to) is executed by a hand-written kernel; torch only owns device memory.  The
engine reads the parameters of an `MM_LLMs` module (modeling.py in this package) and keeps *derived* weights
(fused QKV, interleaved gate/up, permuted conv filters, bf16 shadows) in a cache keyed by parameter version, so
in-place weight updates are picked up.

Data layout in HBM: activations are bf16, token-major `(tokens, channels)` with the residual stream updated in
place by GEMM epilogues; all contractions accumulate in fp32 (registers); scores of the alignment
cross-attention are fp32.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch

from . import lora, ops, quant

BF16 = torch.bfloat16


def ADT():
    """The 16-bit storage dtype of the model being run (set per call by Engine._set_format): bf16, or fp16 for an fp16 model."""
    return ops.ACT()


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class KVCache:
    """The generate branch's per-layer K / V cache, 16-bit: one (B, t_max, 2, E) tensor per layer in the activation format.

    The cache format is decided here and nowhere else: the decoder loop asks its cache to append the prefill's (or a wide
    decode step's) k / v rows, for the decode tail's keywords, and for a decode step's attention over it."""

    def __init__(self, layers):
        self.layers = layers

    @classmethod
    def allocate(cls, B: int, t_max: int, n_layers: int, E: int, dev) -> "KVCache":
        return cls([torch.zeros((B, t_max, 2, E), device=dev, dtype=ADT()) for _ in range(n_layers)])

    def append(self, i: int, qkv: torch.Tensor, B: int, T: int, pos0: int, t0_dev: Optional[torch.Tensor]) -> None:
        ops.kv_append(qkv, B, T, self.layers[i], pos0, t0_dev)

    def tail_kw(self, i: int) -> dict:
        """Keywords of the THIN_QKV decode tail that writes this layer's slot."""
        return dict(cache=self.layers[i])

    def attend(self, i: int, q: torch.Tensor, T: int, kmask, pos0: int, pos_dev: Optional[torch.Tensor], scale: float):
        """A decode step's attention of q (B, T, H, hd) over keys [0, pos0 + T), or [0, pos_dev[1]) when pos_dev is given
        (the whole capacity is handed over; the kernel reads the valid length)."""
        H, hd = q.shape[2], q.shape[3]
        if pos_dev is not None:
            kv = self.layers[i].unflatten(-1, (H, hd))
            return ops.attention(q, kv[:, :, 0], kv[:, :, 1], scale=scale, causal=False, key_mask=kmask, tk_dev=pos_dev[1:2])
        kv = self.layers[i][:, : pos0 + T].unflatten(-1, (H, hd))  # (B, Tk, 2, H, hd) view of the cache
        return ops.attention(q, kv[:, :, 0], kv[:, :, 1], scale=scale, causal=False, key_mask=kmask)


class KVCacheInt8(KVCache):
    """The int8 KV cache (Engine.enable_int8_kv_cache): per layer, int8 values `kq` (B, t_max, 2, E), indexed as the 16-bit
    cache, and fp32 scales `ks` (B, 2, H, t_max), one per (token, head) key or value vector of 128 elements:
    s = fp32(max |v|) / 127, q = clamp(rint(v / s), -127, 127), q = 0 where s = 0, for v as the 16-bit cache would hold it.
    A decode step's attention runs mm_attn_decode_i8 on the dequantized q * s."""

    def __init__(self, kq, ks):
        super().__init__(kq)
        self.ks = ks

    @classmethod
    def allocate(cls, B: int, t_max: int, n_layers: int, E: int, dev) -> "KVCacheInt8":
        return cls([torch.zeros((B, t_max, 2, E), device=dev, dtype=torch.int8) for _ in range(n_layers)],
                   [torch.zeros((B, 2, E // 128, t_max), device=dev, dtype=torch.float32) for _ in range(n_layers)])

    def append(self, i, qkv, B, T, pos0, t0_dev):
        ops.kv_append_i8(qkv, B, T, self.layers[i], self.ks[i], pos0, t0_dev)

    def tail_kw(self, i):
        return dict(cache=self.layers[i], cache_scale=self.ks[i])

    def attend(self, i, q, T, kmask, pos0, pos_dev, scale):
        assert T == 1
        if pos_dev is not None:
            return ops.attention_decode_i8(q, self.layers[i], self.ks[i], scale=scale, tk_dev=pos_dev[1:2], key_mask=kmask)
        return ops.attention_decode_i8(q, self.layers[i], self.ks[i], scale=scale, Tk=pos0 + T, key_mask=kmask)


class Engine:
    def __init__(self, model):
        self.m = model
        self._cache: Dict[str, Tuple[tuple, object]] = {}
        self._rope: Dict[Tuple[int, int, str], Tuple[torch.Tensor, torch.Tensor]] = {}
        self._pe: Dict[Tuple[int, int, str], torch.Tensor] = {}
        self._zeros: Dict[Tuple[int, str], torch.Tensor] = {}
        self._graphs: Dict[tuple, tuple] = {}
        self._decode: Dict[tuple, dict] = {}  # KV buffers + captured decode step per (batch, capacity, device)
        self._side: Dict[str, torch.cuda.Stream] = {}
        # Whisper tower on a side stream next to the CLIP tower(s): both towers' GEMMs are persistent one-CTA-per-SM
        # kernels, two of them cannot co-reside, so only launch tails overlap while the late-starting CTAs stretch the static
        # tile schedule.  Off by default; kept as a tested option.
        self.overlap_encoders = False
        # Stream-K tail in the LLaMA GEMMs (a partial last wave of tiles is split along K over all SMs): matters at small
        # per-GPU batch (e.g. 1088 tiles on 132 SMs -> 8.2 waves), a no-op when the tile count fills the waves.
        self.streamk = True
        self._sk_ws: Dict[str, torch.Tensor] = {}
        self._graphs_on = False
        self.kv_int8 = False  # generate keeps its KV cache in int8 (enable_int8_kv_cache)
        self.align_max_rows = None  # test hook: cap on query rows per alignment chunk (default: ~2 GiB of fp32 scores)

    # ------------------------------------------------------------------------------------------------ weight cache
    @staticmethod
    def _stamp(*params) -> tuple:
        return tuple((p.data_ptr(), p._version, p.dtype) for p in params)

    def drop_derived(self) -> None:
        """Forget every derived weight, captured forward graph and decode state (the parameters were replaced)."""
        self._cache.clear()
        self._graphs.clear()
        self._decode.clear()

    def derived(self, key: str, params, fn):
        st = self._stamp(*params)
        hit = self._cache.get(key)
        if hit is not None and hit[0] == st:
            return hit[1]
        with torch.no_grad():
            val = fn()
        self._cache[key] = (st, val)
        return val

    def w16(self, p: torch.Tensor, key: str) -> torch.Tensor:
        """fp16 copy of a parameter for the fp16 alignment chain: the bf16 value converted exactly (values below fp16's
        normal range lose bits, values above 65504 saturate — neither occurs for weights / embeddings)."""
        self.w(p, key)  # device / dtype checks
        if p.dtype == torch.float16:
            return p.detach()  # an fp16 model already is in the chain's format
        return self.derived("f16:" + key, [p], lambda: p.detach().to(torch.bfloat16).to(torch.float16))

    def set_format(self) -> None:
        """Choose the 16-bit storage format for this call from the model's dtype: an fp16 model (the reference's own
        precision: train.sh `--fp16 True`, llm_trainer.py:366-368 `.half()`) is computed in fp16 — 11-bit significands, the
        storage rounding of every activation is 8x smaller than bf16's; bf16 and fp32 models are computed in bf16 (fp32
        parameters through bf16 shadows).  Sets both the Python-side dtype and the kernel library's thread-local format."""
        dt = self.m.llm.model.embed_tokens.weight.dtype
        ops.set_act_format(torch.float16 if dt == torch.float16 else torch.bfloat16)

    def w(self, p: torch.Tensor, key: str) -> torch.Tensor:
        """CUDA view of a parameter in the activation format (the parameter itself when it already has that dtype)."""
        if not p.is_cuda:
            raise RuntimeError(
                "macaw_b200: model parameters live on the CPU; move the model to a CUDA device "
                "(there is no CPU execution path)")
        if p.dtype == ADT():
            return p.detach()
        return self.derived("shadow:" + key, [p], lambda: p.detach().to(ADT()))

    def zeros(self, n: int, dev) -> torch.Tensor:
        k = (n, str(dev))
        z = self._zeros.get(k)
        if z is None:
            z = torch.zeros((1, n), device=dev, dtype=ADT())
            self._zeros[k] = z
        return z

    # ------------------------------------------------------------------------------------------------ generic blocks
    def _self_attn_block(self, x, B, T, D, H, ln1, wqkv, bqkv, wo, bo, ln2, fc1, fc2, act, eps, scale):
        """Pre-LN encoder layer (CLIP: modeling_clip.py CLIPEncoderLayer; Whisper: modeling_whisper.py WhisperEncoderLayer)."""
        hd = D // H
        h = ops.layernorm(x, ln1[0], ln1[1], eps)
        qkv = ops.linear(h, wqkv, bqkv).view(B, T, 3, H, hd)
        a = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], scale=scale)
        ops.linear(a.view(B * T, D), wo, bo, residual=x, out=x)
        h = ops.layernorm(x, ln2[0], ln2[1], eps)
        f = ops.linear(h, fc1[0], fc1[1], act=act)
        ops.linear(f, fc2[0], fc2[1], residual=x, out=x)
        return x

    # ------------------------------------------------------------------------------------------------ CLIP
    def clip_tokens(self, images: torch.Tensor, which: str) -> torch.Tensor:
        self.set_format()
        return self._clip_tokens(images, which)

    def _clip_tokens(self, images: torch.Tensor, which: str) -> torch.Tensor:
        """visual_projection(vision_model(images)[0])[:, 1:, :] (reference modeling.py:1092 / :1073) -> (n_img, 256, P).

        CLS rows are skipped by the projection GEMM itself (A starts at row 1 of every image)."""
        ops.TAG = "clip"
        clip = getattr(self.m, which)
        vm = clip.vision_model
        cfg = clip.config.vision_config
        D, H, p = cfg.hidden_size, cfg.num_attention_heads, cfg.patch_size
        eps = cfg.layer_norm_eps
        act = {"quick_gelu": ops.ACT_QUICK_GELU, "gelu": ops.ACT_GELU}[cfg.hidden_act]
        n_img = images.shape[0]
        G = (images.shape[2] // p) * (images.shape[3] // p)
        T = G + 1
        dev = images.device
        kp = _round_up(3 * p * p, 64)
        pre = which + ".vision_model."
        emb = vm.embeddings

        def pack_patch():
            wt = emb.patch_embedding.weight.detach().to(ADT()).reshape(D, -1)
            out = torch.zeros((D, kp), device=dev, dtype=ADT())
            out[:, : wt.shape[1]] = wt
            return out

        w_patch = self.derived(pre + "patch", [emb.patch_embedding.weight], pack_patch)
        pos = self.w(emb.position_embedding.weight, pre + "pos")
        if T != pos.shape[0] or images.shape[1] != 3:  # HF CLIPVisionEmbeddings raises on a size mismatch
            raise ValueError(f"Input image size ({images.shape[2]}*{images.shape[3]}) doesn't match model "
                             f"({cfg.image_size}*{cfg.image_size}).")
        cls = self.w(emb.class_embedding, pre + "cls").view(1, D)

        cols = ops.patchify(images, p, kp)  # (n_img * G, kp)
        x = torch.empty((n_img, T, D), device=dev, dtype=ADT())
        # patch embedding + position embedding, written to rows 1..G of every image
        ops.gemm_raw(M=G, N=D, K=kp, batch=n_img, A=cols.data_ptr(), lda=kp, a_bs=G * kp, B=w_patch.data_ptr(), ldb=kp,
                     b_bs=0, Cout=x.data_ptr() + D * 2, ldc=D, c_bs=T * D, residual=pos.data_ptr() + D * 2, ldr=D, r_bs=0)
        # CLS row = class_embedding + pos[0]
        ops.add_rows(cls.expand(n_img, D), pos[:1], x[:, 0, :])
        x2 = x.view(n_img * T, D)
        x2 = ops.layernorm(x2, self.w(vm.pre_layrnorm.weight, pre + "pln.w"), self.w(vm.pre_layrnorm.bias, pre + "pln.b"),
                           eps)
        for i, l in enumerate(vm.encoder.layers):
            k = f"{pre}l{i}."
            sa = l.self_attn
            wqkv = self.derived(k + "wqkv", [sa.q_proj.weight, sa.k_proj.weight, sa.v_proj.weight],
                                lambda sa=sa: torch.cat([sa.q_proj.weight, sa.k_proj.weight, sa.v_proj.weight], 0).detach().to(ADT()).contiguous())
            bqkv = self.derived(k + "bqkv", [sa.q_proj.bias, sa.k_proj.bias, sa.v_proj.bias],
                                lambda sa=sa: torch.cat([sa.q_proj.bias, sa.k_proj.bias, sa.v_proj.bias], 0).detach().to(ADT()).contiguous())
            x2 = self._self_attn_block(
                x2, n_img, T, D, H,
                (self.w(l.layer_norm1.weight, k + "ln1w"), self.w(l.layer_norm1.bias, k + "ln1b")),
                wqkv, bqkv, self.w(sa.out_proj.weight, k + "wo"), self.w(sa.out_proj.bias, k + "bo"),
                (self.w(l.layer_norm2.weight, k + "ln2w"), self.w(l.layer_norm2.bias, k + "ln2b")),
                (self.w(l.mlp.fc1.weight, k + "fc1w"), self.w(l.mlp.fc1.bias, k + "fc1b")),
                (self.w(l.mlp.fc2.weight, k + "fc2w"), self.w(l.mlp.fc2.bias, k + "fc2b")),
                act, eps, (D // H) ** -0.5)
        wp = self.w(clip.visual_projection.weight, which + ".vproj")
        P = wp.shape[0]
        tok = torch.empty((n_img, G, P), device=dev, dtype=ADT())
        ops.gemm_raw(M=G, N=P, K=D, batch=n_img, A=x2.data_ptr() + D * 2, lda=D, a_bs=T * D, B=wp.data_ptr(), ldb=D, b_bs=0,
                     Cout=tok.data_ptr(), ldc=P, c_bs=G * P)
        return tok

    # ------------------------------------------------------------------------------------------------ Whisper
    def whisper_encode(self, mel: torch.Tensor) -> torch.Tensor:
        """audio_encoder.encoder(mel)[0] (reference modeling.py:1081-1083) -> (B, 1500, d_model).

        Both stem convolutions run as GEMMs over overlapping row windows of a time-major, zero-padded buffer
        (no im2col copy): conv1 k=3 s=1 p=1, conv2 k=3 s=2 p=1; GELU and the position embedding ride the epilogues."""
        ops.TAG = "whisper"
        self.set_format()
        enc = self.m.audio_encoder.encoder
        cfg = self.m.audio_encoder.config
        D, H = cfg.d_model, cfg.encoder_attention_heads
        act = {"gelu": ops.ACT_GELU}[cfg.activation_function]
        B, C, Tm = mel.shape
        dev = mel.device
        pre = "audio_encoder.encoder."
        w1 = self.derived(pre + "conv1", [enc.conv1.weight],
                          lambda: enc.conv1.weight.detach().to(ADT()).permute(0, 2, 1).reshape(D, 3 * C).contiguous())
        w2 = self.derived(pre + "conv2", [enc.conv2.weight],
                          lambda: enc.conv2.weight.detach().to(ADT()).permute(0, 2, 1).reshape(D, 3 * D).contiguous())
        xt = ops.transpose_pad(mel, 1)  # (B, Tm + 2, C)
        h1 = torch.empty((B, Tm + 2, D), device=dev, dtype=ADT())
        z = self.zeros(D, dev)
        ops.add_rows(z.expand(B, D), None, h1[:, 0, :])
        ops.add_rows(z.expand(B, D), None, h1[:, Tm + 1, :])
        ops.gemm_raw(M=Tm, N=D, K=3 * C, batch=B, A=xt.data_ptr(), lda=C, a_bs=(Tm + 2) * C, B=w1.data_ptr(), ldb=3 * C, b_bs=0,
                     Cout=h1.data_ptr() + D * 2, ldc=D, c_bs=(Tm + 2) * D, bias=self.w(enc.conv1.bias, pre + "b1").data_ptr(),
                     act=ops.ACT_GELU)
        T = Tm // 2
        pos = self.w(enc.embed_positions.weight, pre + "pos")
        if T != pos.shape[0]:  # HF WhisperEncoder.forward raises on any other mel length; the GEMM reads pos by raw pointer
            raise ValueError(f"Whisper expects the mel input features to be of length {2 * pos.shape[0]}, but found {Tm}. "
                             f"Make sure to pad the input mel features to {2 * pos.shape[0]}.")
        x = torch.empty((B, T, D), device=dev, dtype=ADT())
        ops.gemm_raw(M=T, N=D, K=3 * D, batch=B, A=h1.data_ptr(), lda=2 * D, a_bs=(Tm + 2) * D, B=w2.data_ptr(), ldb=3 * D,
                     b_bs=0, Cout=x.data_ptr(), ldc=D, c_bs=T * D, bias=self.w(enc.conv2.bias, pre + "b2").data_ptr(),
                     act=ops.ACT_GELU, residual=pos.data_ptr(), ldr=D, r_bs=0)
        x2 = x.view(B * T, D)
        for i, l in enumerate(enc.layers):
            k = f"{pre}l{i}."
            sa = l.self_attn
            wqkv = self.derived(k + "wqkv", [sa.q_proj.weight, sa.k_proj.weight, sa.v_proj.weight],
                                lambda sa=sa: torch.cat([sa.q_proj.weight, sa.k_proj.weight, sa.v_proj.weight], 0).detach().to(ADT()).contiguous())
            bqkv = self.derived(k + "bqkv", [sa.q_proj.bias, sa.v_proj.bias],
                                lambda sa=sa: torch.cat([sa.q_proj.bias, torch.zeros_like(sa.q_proj.bias), sa.v_proj.bias], 0).detach().to(ADT()).contiguous())
            x2 = self._self_attn_block(
                x2, B, T, D, H,
                (self.w(l.self_attn_layer_norm.weight, k + "ln1w"), self.w(l.self_attn_layer_norm.bias, k + "ln1b")),
                wqkv, bqkv, self.w(sa.out_proj.weight, k + "wo"), self.w(sa.out_proj.bias, k + "bo"),
                (self.w(l.final_layer_norm.weight, k + "ln2w"), self.w(l.final_layer_norm.bias, k + "ln2b")),
                (self.w(l.fc1.weight, k + "fc1w"), self.w(l.fc1.bias, k + "fc1b")),
                (self.w(l.fc2.weight, k + "fc2w"), self.w(l.fc2.bias, k + "fc2b")),
                act, 1e-5, (D // H) ** -0.5)
        x2 = ops.layernorm(x2, self.w(enc.layer_norm.weight, pre + "lnw"), self.w(enc.layer_norm.bias, pre + "lnb"), 1e-5)
        return x2.view(B, T, D)

    # ------------------------------------------------------------------------------------------------ video-long
    def video_pe(self, L: int, h: int, dev) -> torch.Tensor:
        """Sinusoid table of create_positional_encoding (reference modeling.py:1095-1106), built once per shape on the
        host with the reference's exact fp32 arithmetic (exponent 2*i with i already even) instead of its O(L*h)
        python loop per forward."""
        key = (L, h, str(dev))
        pe = self._pe.get(key)
        if pe is None:
            arg = torch.tensor([-(math.log(10000.0) / h * (2 * i)) for i in range(0, h, 2)], dtype=torch.float32)
            div = torch.exp(arg)
            pos = torch.arange(L, dtype=torch.float32)[:, None]
            t = torch.zeros(L, h, dtype=torch.float32)
            t[:, 0::2] = torch.sin(pos * div)
            t[:, 1::2] = torch.cos(pos * div)
            pe = t.to(ADT()).to(dev)
            self._pe[key] = pe
        return pe

    def encode_video_long(self, videos: torch.Tensor, save: Optional[dict] = None, dropout=None) -> torch.Tensor:
        """reference modeling.py:1070-1079 -> (B, F*256, P).  `save` (training step) receives the activations of the
        video_long_self_attention block (its input xp, the fused qkv buffer with the two synthetic key rows, the attention
        output) for the backward pass; `dropout` = (p, seed_dev, sid): its attention dropout (train() mode) — the
        probabilities are then materialised (GEMM -> softmax + Philox mask -> GEMM) instead of the flash kernel."""
        m = self.m
        F_ = m.config.n_frames
        frames = videos.reshape(-1, *videos.shape[-3:])
        tok = self.clip_tokens(frames, "video_encoder")  # (B*F, G, P)
        B = frames.shape[0] // F_
        G, P = tok.shape[1], tok.shape[2]
        N = F_ * G
        dev = videos.device
        ops.TAG = "video_long"
        x = tok.view(B * N, P)
        pe = self.video_pe(N, P, dev)
        xp = torch.empty_like(x)
        ops.add_rows(x, pe, xp)
        mha = m.video_long_self_attention
        H = mha.num_heads
        hd = P // H
        pre = "video_long_self_attention."
        w_in = self.w(mha.in_proj_weight, pre + "win")
        b_in = self.w(mha.in_proj_bias, pre + "bin")
        qkv = torch.empty((B, N + 2, 3 * P), device=dev, dtype=ADT())
        ops.gemm_raw(M=N, N=3 * P, K=P, batch=B, A=xp.data_ptr(), lda=P, a_bs=N * P, B=w_in.data_ptr(), ldb=P, b_bs=0,
                     Cout=qkv.data_ptr(), ldc=3 * P, c_bs=(N + 2) * 3 * P, bias=b_in.data_ptr())
        # synthetic keys: row N = (bias_k, bias_v) appended un-projected, row N+1 = zeros (functional.py:6531-6537, 6585-6602)
        bk = self.w(mha.bias_k, pre + "bk").view(1, P)
        bv = self.w(mha.bias_v, pre + "bv").view(1, P)
        z = self.zeros(P, dev)
        ops.add_rows(bk.expand(B, P), None, qkv[:, N, P:2 * P])
        ops.add_rows(bv.expand(B, P), None, qkv[:, N, 2 * P:])
        ops.add_rows(z.expand(B, P), None, qkv[:, N + 1, P:2 * P])
        ops.add_rows(z.expand(B, P), None, qkv[:, N + 1, 2 * P:])
        q5 = qkv.view(B, N + 2, 3, H, hd)
        if dropout is not None and save is not None and float(dropout[0]) > 0.0:
            a = ops.attention_train_fwd(q5[:, :N, 0], q5[:, :, 1], q5[:, :, 2], scale=hd ** -0.5, dropout=dropout)
        else:
            dropout = None
            a = ops.attention(q5[:, :N, 0], q5[:, :, 1], q5[:, :, 2], scale=hd ** -0.5)
        out = ops.linear(a.view(B * N, P), self.w(mha.out_proj.weight, pre + "wo"), self.w(mha.out_proj.bias, pre + "bo"))
        if save is not None:
            save.update(xp=xp, qkv=qkv, a=a, B=B, N=N, P=P, H=H, hd=hd, dropout=dropout)
        return out.view(B, N, P)

    # ------------------------------------------------------------------------------------------------ alignment
    def align(self, feats: torch.Tensor, name: str, table: torch.Tensor, prefix: torch.Tensor, row_off: int,
              table16: Optional[torch.Tensor] = None, save: Optional[dict] = None, dropout=None) -> int:
        """One modality of reference modeling.py:982-987 / 999-1008 / 1022-1026 in ABSORBED form (SURVEY.md §7):
        the keys/values are never projected — q is pushed through W_k per head and both big contractions
        (scores = q~ . table^T over E, ctx~ = P . table over V) run inside ONE fused kernel (mm_align_fwd) that streams
        tiles of the raw embedding table through TMA; neither the scores nor a softmax pass ever touch HBM in fp32.

        Precision: the whole chain runs in fp16 x fp16 -> fp32 (11-bit significand; one stored stage costs 1.4e-4
        norm-wise, bf16 1.1e-3) on exact fp16 copies of the bf16 weights / table, so the block's error is dominated by
        the single bf16 rounding of its output.

        feats (B, N, C) bf16 with unit channel stride and row stride C (sample stride free); writes the Lq aligned
        rows into prefix[:, row_off : row_off + Lq] and returns Lq.

        dropout = (p, seed_dev, sid) (training step only, with `save`): the MHA's attention dropout (modeling.py:879) on the
        (V + 2)-key probabilities — the fused kernel's fp16 P' is masked (Philox, regenerated in the backward pass) and the
        P . table contraction is redone on the masked probabilities."""
        ops.TAG = "align.proj"
        F16 = torch.float16
        m = self.m
        conv = getattr(m, f"project_{name}")
        lin = getattr(m, f"transform_{name}_to_hidden")
        mha = getattr(m, f"{name}_align_attention")
        B, N, C = feats.shape
        assert feats.stride(2) == 1 and feats.stride(1) == C
        feats_bf = feats.contiguous()
        feats = feats_bf if feats_bf.dtype == F16 else ops.cast_f16(feats_bf)
        if table16 is None:  # stand-alone use (tests / tools): exact fp16 copy of the given table
            table16 = self.derived("align.table16", [table], lambda: table.detach().to(F16))
        assert table16.shape == table.shape and table16.dtype == F16
        kk, ss = conv.kernel_size[0], conv.stride[0]
        Lq = (N - kk) // ss + 1
        Nq = B * Lq
        E = table.shape[1]
        V = table.shape[0]
        H = mha.num_heads
        hd = E // H
        dev = feats.device
        pre = f"{name}_align."
        f16 = dict(a_fp16=True, b_fp16=True)
        # ---- Conv1d over the token axis == GEMM on overlapping row windows (window = kk*C contiguous elements), split over K
        wc = self.derived(pre + "conv", [conv.weight],
                          lambda: conv.weight.detach().to(ADT()).to(F16).permute(0, 2, 1).reshape(C, kk * C).contiguous())
        K = kk * C
        S = 1
        for cand in (16, 12, 9, 8, 6, 4, 3, 2):
            if K % (cand * 64) == 0:
                S = cand
                break
        Kc = K // S
        part = torch.empty((S, Nq, C), device=dev, dtype=torch.float32)
        ops.gemm_raw(M=Lq, N=C, K=Kc, batch=S, batch2=B, A=feats.data_ptr(), lda=ss * C, a_bs=Kc, a_bs2=feats.stride(0),
                     B=wc.data_ptr(), ldb=K, b_bs=Kc, b_bs2=0, Cout=part.data_ptr(), ldc=C, c_bs=Nq * C, c_bs2=Lq * C,
                     c_fp32=True, **f16)
        y = torch.empty((Nq, C), device=dev, dtype=F16)
        ops.splitk_reduce(part, self.w(conv.bias, pre + "convb"), y)
        # ---- Linear C -> E, then the MHA query projection
        z = ops.linear(y, self.w16(lin.weight, pre + "lw"), self.w(lin.bias, pre + "lb"), out_dtype=F16)
        w_in = self.w16(mha.in_proj_weight, pre + "win")
        b_in = self.w(mha.in_proj_bias, pre + "bin")
        q = ops.linear(z, w_in[:E], b_in[:E], out_dtype=F16)  # (Nq, E); the 1/sqrt(hd) scale is applied downstream (alpha)
        w_k, w_v = w_in[E:2 * E], w_in[2 * E:]
        bk2 = self.derived(pre + "bk2", [mha.in_proj_bias, mha.bias_k],
                           lambda: torch.stack([mha.in_proj_bias.detach()[E:2 * E].to(ADT()),
                                                mha.bias_k.detach().reshape(E).to(ADT())], 0).to(F16).contiguous())
        b_v = b_in[2 * E:]
        bias_v = self.w(mha.bias_v, pre + "biasv").view(E)
        scale = 1.0 / math.sqrt(hd)
        Vp = _round_up(V, 8)
        ctx = torch.empty((Nq, E), device=dev, dtype=F16)
        # bound the fp16 probability scratch (R x V) to ~2 GiB by chunking query rows
        max_nq = max(1, (1 << 31) // (H * Vp * 2))
        if self.align_max_rows:
            max_nq = min(max_nq, int(self.align_max_rows))
        for n0 in range(0, Nq, max_nq):
            n1 = min(Nq, n0 + max_nq)
            nq = n1 - n0
            R = H * nq
            qs = q[n0:n1]
            # per-row constants: q_h . b_k[h] (added to every real key) and q_h . bias_k[h] (the bias_k key's score)
            stats = torch.empty((H, nq, 2), device=dev, dtype=torch.float32)
            ops.gemm_raw(M=nq, N=2, K=hd, batch=H, A=qs.data_ptr(), lda=E, a_bs=hd, B=bk2.data_ptr(), ldb=E, b_bs=hd,
                         Cout=stats.data_ptr(), ldc=2, c_bs=nq * 2, c_fp32=True, alpha=scale, **f16)
            # q~[h] = (q_h / sqrt(hd)) W_k[h]   (B operand = W_k rows of head h, N-contiguous -> MN-major UMMA descriptor)
            qt = torch.empty((H, nq, E), device=dev, dtype=F16)
            ops.gemm_raw(M=nq, N=E, K=hd, batch=H, A=qs.data_ptr(), lda=E, a_bs=hd, B=w_k.data_ptr(), ldb=E, b_bs=hd * E,
                         b_mn_major=True, Cout=qt.data_ptr(), ldc=E, c_bs=nq * E, alpha=scale, c_fp16=True, **f16)
            # ctx~ = softmax(q~ . table^T + bias terms)[:, :V] . table — the fused kernel (both table contractions)
            keep = {} if save is not None else None
            ctxt, psum, pext = ops.align_fused(table16, qt.view(R, E), stats.view(R, 2), keep=keep)
            if save is not None:
                if nq != Nq:
                    raise NotImplementedError("macaw_b200 training: the alignment block must fit one row chunk")
                save.update(keep)
                save.update(pext_raw=pext, dropout=None)
                if dropout is not None and float(dropout[0]) > 0.0:
                    ops.TAG = "align.dropout"
                    Pm, rs, psum, pext = ops.align_dropout_fwd(keep["P"], keep["inv_l"], pext, V, dropout)
                    ops.gemm_raw(M=R, N=E, K=V, A=Pm.data_ptr(), lda=Vp, B=table16.data_ptr(), ldb=table16.stride(0),
                                 b_mn_major=True, Cout=ctxt.data_ptr(), ldc=E, row_scale=rs.data_ptr(), c_fp16=True, **f16)
                    del Pm
                    save.update(dropout=dropout)
                save.update(feats=feats_bf, y=y, z=z, q=q, stats=stats, qt=qt, ctxt=ctxt, psum=psum, pext=pext, ctx=ctx,
                            B=B, N=N, C=C, Lq=Lq, kk=kk, ss=ss, H=H, hd=hd, row_off=row_off)
            # ctx[:, h] = ctx~[h] W_v[h]^T + (sum_real P) b_v[h] + P_bias bias_v[h]   (value-side bias terms in the epilogue)
            cs = ctx[n0:n1]
            ops.TAG = "align.proj"
            ops.gemm_raw(M=nq, N=hd, K=E, batch=H, A=ctxt.data_ptr(), lda=E, a_bs=nq * E, B=w_v.data_ptr(), ldb=E,
                         b_bs=hd * E, Cout=cs.data_ptr(), ldc=E, c_bs=hd, c_fp16=True, **f16,
                         bias=b_v.data_ptr(), bias_bs=hd, bias_rs=psum.data_ptr(), bias2=bias_v.data_ptr(),
                         bias2_rs=pext.data_ptr())
        # ---- out_proj straight into the prefix block of every sample
        Ptot = prefix.shape[1]
        ops.gemm_raw(M=Lq, N=E, K=E, batch=B, A=ctx.data_ptr(), lda=E, a_bs=Lq * E,
                     B=self.w16(mha.out_proj.weight, pre + "wo").data_ptr(), ldb=E, b_bs=0,
                     Cout=prefix.data_ptr() + row_off * E * 2, ldc=E, c_bs=Ptot * E,
                     bias=self.w(mha.out_proj.bias, pre + "bo").data_ptr(), **f16)
        return Lq

    @staticmethod
    def align_len(n_tokens: int, kernel: int, stride: int) -> int:
        return (n_tokens - kernel) // stride + 1

    # ------------------------------------------------------------------------------------------------ input preparation
    def _to_dev_bf16(self, t: torch.Tensor, dev) -> torch.Tensor:
        if t.device != dev:
            t = t.to(dev, non_blocking=True)
        if t.dtype != ADT():
            t = t.to(ADT())
        return t.contiguous()

    DROPOUT_SID = {"image": 1, "audio": 2, "video": 3, "video_long": 4}  # Philox stream id of each dropout site

    def prepare_inputs(self, inputs: dict, save: Optional[dict] = None, dropout_seed: Optional[torch.Tensor] = None):
        """MM_LLMs.prepare_inputs_for_generation (reference modeling.py:965-1048).  `save` (training step): receives the
        alignment activations of every modality, keyed by modality name, for the backward pass.  `dropout_seed` (training
        step, train() mode): device int64 seed -> the attention dropout of the MHAs (modeling.py:879) is applied."""
        m = self.m
        self.set_format()
        table = self.w(m.llm.model.embed_tokens.weight, "llm.embed")
        dev = table.device
        E = table.shape[1]
        ids = inputs["input_ids"]
        V_rows = table.shape[0]
        for k in ("input_ids", "image_starts", "image_ends", "audio_starts", "audio_ends", "video_starts", "video_ends"):
            t = inputs.get(k)
            # nn.Embedding raises on out-of-range ids; the gather kernel clamps, so host-resident ids are validated here
            # (device-resident ids would need a sync: they stay clamped, as documented in include/macaw_b200.h)
            if isinstance(t, torch.Tensor) and not t.is_cuda and t.numel() > 0:
                lo, hi = int(t.min()), int(t.max())
                if lo < 0 or hi >= V_rows:
                    raise IndexError(f"{k}: token id out of range for the {V_rows}-row embedding table (min {lo}, max {hi}); "
                                     f"call model.llm.resize_token_embeddings(len(tokenizer)) first")
        ids = ids.to(dev)
        B, L = ids.shape
        feats = {}
        mel = self._to_dev_bf16(inputs["audios"], dev) if inputs.get("audios") is not None else None
        side = None
        if mel is not None and self.overlap_encoders and (inputs.get("images") is not None or inputs.get("videos") is not None):
            # The Whisper tower is independent of the CLIP tower(s): run it on a side stream so its short-K GEMMs fill the
            # SMs the other tower's 108..144-tile launches leave idle (the two towers' kernels interleave; under CUDA-graph
            # capture the fork / join becomes graph edges).  Joined before the alignment blocks.
            main = torch.cuda.current_stream(dev)
            side = self._side.get(str(dev))
            if side is None:
                side = self._side[str(dev)] = torch.cuda.Stream(device=dev)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                feats["audio"] = self.whisper_encode(mel)
            mel.record_stream(side)
        if inputs.get("images") is not None:
            feats["image"] = self.clip_tokens(self._to_dev_bf16(inputs["images"], dev), "image_encoder")
        if mel is not None and side is None:
            feats["audio"] = self.whisper_encode(mel)
        if inputs.get("videos") is not None:
            mha_v = m.video_long_self_attention
            feats["video"] = self.encode_video_long(
                self._to_dev_bf16(inputs["videos"], dev), save=None if save is None else save.setdefault("video_long", {}),
                dropout=None if dropout_seed is None else (float(mha_v.dropout), dropout_seed, self.DROPOUT_SID["video_long"]))
        if side is not None:
            torch.cuda.current_stream(dev).wait_stream(side)
            feats["audio"].record_stream(torch.cuda.current_stream(dev))
            self.set_format()
        # final layout [BOS, <image> img </image>, <audio> aud </audio>, <video> vid </video>, text[1:]]: each block is
        # spliced right after BOS in the order video, audio, image (reference modeling.py:978-1034), so image ends up first
        lens = {}
        for name in ("image", "audio", "video"):
            if name in feats:
                conv = getattr(m, f"project_{name}")
                lens[name] = self.align_len(feats[name].shape[1], conv.kernel_size[0], conv.stride[0])
        n_prefix = sum(v + 2 for v in lens.values())
        if "video" in feats:
            self._video_long_len = feats["video"].shape[1]  # tokens of video_long_self_attention (frames x patches)
        self.last_lens = dict(lens)  # aligned rows per modality of the most recent call (the training step maps prefix rows to token ids)
        prefix = None
        if n_prefix > 0:
            prefix = torch.empty((B, n_prefix, E), device=dev, dtype=ADT())
            off = 0
            for name in ("image", "audio", "video"):
                if name not in feats:
                    continue
                Lq = lens[name]
                ops.embed_gather(table, inputs[f"{name}_starts"].to(dev), out=prefix[:, off, :])
                sv = None
                if save is not None:
                    sv = save.setdefault(name, {})
                drop = None
                if dropout_seed is not None and sv is not None:
                    drop = (float(getattr(m, f"{name}_align_attention").dropout), dropout_seed, self.DROPOUT_SID[name])
                got = self.align(feats[name], name, table, prefix, off + 1,
                                 self.w16(m.llm.model.embed_tokens.weight, "llm.embed"), save=sv, dropout=drop)
                assert got == Lq
                ops.embed_gather(table, inputs[f"{name}_ends"].to(dev), out=prefix[:, off + 1 + Lq, :])
                off += Lq + 2
        text = ops.embed_gather(table, ids).view(B, L, E)
        mask_in = inputs["attention_mask"].to(dev) if "attention_mask" in inputs else None
        labels_in = inputs["labels"].to(dev) if inputs.get("labels") is not None else None
        return ops.splice_prefix(text, prefix, mask_in, labels_in)

    # ------------------------------------------------------------------------------------------------ LLaMA
    def rope_tables(self, T: int, hd: int, dev):
        """cos/sin (T, hd/2) fp32.  Always rebuilt from the closed form (base 1e4, reference modeling.py:97-107): the
        reference caches cos/sin at construction in fp32, so a later `.half()` / `.to(bf16)` of the `inv_freq`
        buffer must not change the angles."""
        key = (T, hd, str(dev))
        t = self._rope.get(key)
        if t is None:
            inv = (1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))).to(dev)
            fr = torch.arange(T, device=dev, dtype=torch.float32)[:, None] * inv[None, :]
            t = (fr.cos().contiguous(), fr.sin().contiguous())
            self._rope[key] = t
        return t

    def _llama_weights(self, i: int, l, E: int, I: int):
        """Derived weights of decoder layer i: fused [q;k;v] and 32-row-interleaved [gate|up], RMSNorm gains folded in
        (fp32 product, one bf16 rounding): RMSNorm(x) W^T = rstd * (x (W diag g)^T)."""
        k = f"llm.l{i}."
        sa, mlp = l.self_attn, l.mlp
        g1, g2 = l.input_layernorm.weight, l.post_attention_layernorm.weight
        # LoRA adapters are folded in: lora.merged_weight is W + s B A in fp32 for an adapted projection (W otherwise)
        wqkv = self.derived(k + "wqkv", lora.weight_params(sa.q_proj) + lora.weight_params(sa.k_proj)
                            + lora.weight_params(sa.v_proj) + [g1],
                            lambda: (torch.cat([lora.merged_weight(sa.q_proj), lora.merged_weight(sa.k_proj),
                                                lora.merged_weight(sa.v_proj)], 0)
                                     * g1.detach().float()[None, :]).to(ADT()).contiguous())
        wgu = self.derived(k + "wgu", lora.weight_params(mlp.gate_proj) + lora.weight_params(mlp.up_proj) + [g2],
                           lambda: torch.stack(
                               [(lora.merged_weight(mlp.gate_proj) * g2.detach().float()[None, :]).to(ADT()).view(I // 32, 32, E),
                                (lora.merged_weight(mlp.up_proj) * g2.detach().float()[None, :]).to(ADT()).view(I // 32, 32, E)], 1)
                           .reshape(2 * I, E).contiguous())
        return wqkv, wgu, self._linear_weight(sa.o_proj, k + "wo"), self._linear_weight(mlp.down_proj, k + "wd")

    def _w8_layer(self, i: int, l):
        """The int8 weights of a quantized decoder layer as fused matrices: [q; k; v] and [gate | up] with their RMSNorm
        gains (applied to the activation rows by the decode GEMM, folded into the rows by the dequantization), o, down."""
        sa, mlp = l.self_attn, l.mlp
        g1 = self.w(l.input_layernorm.weight, f"llm.l{i}.g1")
        g2 = self.w(l.post_attention_layernorm.weight, f"llm.l{i}.g2")
        src = lambda *ms: ([m.weight for m in ms], [m.weight_scale for m in ms])
        return (ops.W8Matrix(*src(sa.q_proj, sa.k_proj, sa.v_proj), gain=g1),
                ops.W8Matrix(*src(mlp.gate_proj, mlp.up_proj), interleave=True, gain=g2),
                ops.W8Matrix(*src(sa.o_proj)), ops.W8Matrix(*src(mlp.down_proj)))

    def _linear_weight(self, lin, key: str) -> torch.Tensor:
        """The weight of a linear layer in the activation format, its LoRA adapter merged in when it carries one."""
        if not lora.is_adapted(lin):
            return self.w(lin.weight, key)
        return self.derived("lora:" + key, lora.weight_params(lin),
                            lambda: lora.merged_weight(lin).to(ADT()).contiguous())

    def _llama_dims(self):
        cfg = self.m.llm.config
        E, H = cfg.hidden_size, cfg.num_attention_heads
        hd = E // H
        if hd != 128:
            raise NotImplementedError(f"macaw_b200: LLaMA head_dim {hd} unsupported (RoPE epilogue is specialised for 128)")
        I = cfg.intermediate_size
        if I % 32 != 0:
            raise NotImplementedError("macaw_b200: intermediate_size must be a multiple of 32")
        return E, H, hd, I, cfg.rms_norm_eps

    def _streamk_ws(self, dev) -> Optional[torch.Tensor]:
        """Stream-K workspace of the LLaMA section on `dev` (its GEMMs run back to back on one stream)."""
        if not self.streamk:
            return None
        ws = self._sk_ws.get(str(dev))
        if ws is None:
            ws = self._sk_ws[str(dev)] = ops.streamk_workspace(dev)
        return ws

    def _llama_layers(self, x: torch.Tensor, *args, **kw):
        ops.STREAMK = self._streamk_ws(x.device)
        try:
            return self._llama_layers_impl(x, *args, **kw)
        finally:
            ops.STREAMK = None

    def _llama_layers_impl(self, x: torch.Tensor, B: int, T: int, kmask, pos0: int = 0, cache=None, t_max: int = 0,
                           pos_dev: Optional[torch.Tensor] = None):
        """The decoder stack on the residual stream x (B*T, E), updated in place.

        pos0 = position of the first row of every sample (0 for prefill, the current length for a decode step).
        With `cache` (a KVCache, or a list of per-layer (B, Tmax, 2, E) 16-bit tensors) the new K/V rows are appended at
        pos0 and, for decode steps (pos0 > 0), attention reads keys/values [0, pos0 + T) from the cache (reference KV-cache
        logic: modeling.py:190-195).
        `pos_dev` (int32 tensor [pos, pos + 1] on the device) replaces pos0 for a decode step whose launches are captured
        in a CUDA graph: RoPE position, cache slot and key count are then read by the kernels themselves."""
        E, H, hd, I, eps = self._llama_dims()
        dev = x.device
        cos, sin = self.rope_tables(max(T, t_max), hd, dev)
        scale = 1.0 / math.sqrt(hd)
        dyn = pos_dev is not None
        if dyn:
            rope = (cos, sin, 1, 2 * E, pos_dev[0:1])
        else:
            rope = (cos, sin, T, 2 * E) if pos0 == 0 else (cos[pos0:], sin[pos0:], 1, 2 * E)
        assert (pos0 == 0 and not dyn) or T == 1
        # Decode step (one new token per sample, at most 64 samples): each GEMM swaps its operands so the weights fill the
        # 128-row MMA tiles, splits K, and ends in ONE tail kernel that also does the neighbouring row-wise work (RoPE +
        # KV-cache write / SwiGLU / residual + next RMSNorm statistic): 9 launches per layer.  Everything else runs the
        # wide GEMMs, whose epilogues apply RoPE, SwiGLU and the residual adds.
        # Either way the RMSNorm statistics ride the GEMM epilogues: the GEMM that WRITES the residual stream (o_proj /
        # down_proj) leaves per-(row, 32-column) sums of squares of the stored values, the GEMM that CONSUMES it (QKV /
        # gate-up / lm_head) derives rsqrt(mean(x^2) + eps) from them — no separate pass over the stream after the first
        # layer's input.
        M = x.shape[0]
        if cache is not None and not isinstance(cache, KVCache):
            cache = KVCache(cache)
        decode = cache is not None and T == 1 and B <= 64
        ss_attn = torch.empty((M, E // 32), device=dev, dtype=torch.float32)
        ss_mlp = torch.empty((M, E // 32), device=dev, dtype=torch.float32)
        # int8 decoder (quant.py): decode steps run the int8 GEMM ahead of the same tails; everything else dequantizes one
        # layer at a time into one scratch buffer and runs the 16-bit GEMMs below unchanged.  An FP8 decoder has its own loop.
        fmt = quant.quant_format(self.m)
        if fmt == "fp8":
            return self._llama_layers_fp8(x, B, T, kmask, pos0, cache, dyn, pos_dev, rope, decode, ss_attn, ss_mlp)
        w8 = fmt == "int8"
        thin = ops.linear_w8_thin_fused if w8 else ops.linear_thin_fused
        if w8 and not decode:
            scratch = torch.empty((3 * E + 2 * I + E) * E + E * I, device=dev, dtype=ADT())
            views, off = [], 0
            for n, k in ((3 * E, E), (2 * I, E), (E, E), (E, I)):
                views.append(scratch[off:off + n * k].view(n, k))
                off += n * k
        for i, l in enumerate(self.m.llm.model.layers):
            if w8:
                mats = self._w8_layer(i, l)
                wqkv, wgu, wo, wd = mats if decode else [ops.dequant_rows(m, out=v) for m, v in zip(mats, views)]
            else:
                wqkv, wgu, wo, wd = self._llama_weights(i, l, E, I)
            rs_kw = dict(row_scale=ops.rms_rstd(x, eps)) if i == 0 else dict(rms_from=(ss_mlp, eps))
            if decode:
                qkv = thin(x, wqkv, ops.THIN_QKV, rope=(rope[0], rope[1], rope[4] if len(rope) > 4 else None),
                           t0=pos0, t0_dev=pos_dev[0:1] if dyn else None, **cache.tail_kw(i), **rs_kw)
            else:
                qkv = ops.linear(x, wqkv, epi=ops.EPI_ROPE, rope=rope, **rs_kw)
                if cache is not None:
                    cache.append(i, qkv, B, T, pos0, pos_dev[0:1] if dyn else None)
            a = self._attention(qkv.view(B, T, 3, H, hd), T, i, kmask, pos0, cache, dyn, pos_dev, scale)
            if decode:
                thin(a.view(B * T, E), wo, ops.THIN_RES, residual=x, out=x, sumsq_out=ss_attn)
                g = thin(x, wgu, ops.THIN_SWIGLU, rms_from=(ss_attn, eps))
                thin(g, wd, ops.THIN_RES, residual=x, out=x, sumsq_out=ss_mlp)
            else:
                ops.linear(a.view(B * T, E), wo, residual=x, out=x, sumsq_out=ss_attn)
                g = ops.linear(x, wgu, epi=ops.EPI_SWIGLU, rms_from=(ss_attn, eps))
                ops.linear(g, wd, residual=x, out=x, sumsq_out=ss_mlp)
        self._last_ss = None if decode else ss_mlp  # statistics of the final residual stream (consumed by _lm_head)
        return x

    def _attention(self, q5, T, i, kmask, pos0, cache, dyn, pos_dev, scale):
        """The decoder's attention over the new rows' q / k / v (prefill) or the KV cache (decode step)."""
        if pos0 == 0 and not dyn:
            return ops.attention(q5[:, :, 0], q5[:, :, 1], q5[:, :, 2], scale=scale, causal=True, key_mask=kmask)
        return cache.attend(i, q5[:, :, 0], T, kmask, pos0, pos_dev if dyn else None, scale)

    def _llama_layers_fp8(self, x, B, T, kmask, pos0, cache, dyn, pos_dev, rope, decode, ss_attn, ss_mlp):
        """_llama_layers_impl on an FP8 decoder (quant.quantize_llm_fp8).  Decode steps with up to 64 samples stream the
        e4m3 weights through mm_gemm_e4m3_thin (activations not quantized) ahead of the 16-bit path's tails.  Everything
        else quantizes each GEMM input per row (x g1, the attention output, x g2, the SwiGLU output: the RMSNorm gain is
        applied before quantizing, its row statistic in the epilogue as on the 16-bit path) and runs mm_gemm_e4m3_fwd with
        the same epilogues."""
        E, H, hd, I, eps = self._llama_dims()
        scale = 1.0 / math.sqrt(hd)
        for i, l in enumerate(self.m.llm.model.layers):
            wqkv, wgu, wo, wd = self._w8_layer(i, l)
            rs_kw = dict(row_scale=ops.rms_rstd(x, eps)) if i == 0 else dict(rms_from=(ss_mlp, eps))
            if decode:
                thin = ops.linear_w8_thin_fused
                qkv = thin(x, wqkv, ops.THIN_QKV, rope=(rope[0], rope[1], rope[4] if len(rope) > 4 else None),
                           t0=pos0, t0_dev=pos_dev[0:1] if dyn else None, **cache.tail_kw(i), **rs_kw)
            else:
                qkv = ops.linear_e4m3(*ops.quantize_rows_e4m3(x, wqkv.gain), wqkv, epi=ops.EPI_ROPE, rope=rope, **rs_kw)
                if cache is not None:
                    cache.append(i, qkv, B, T, pos0, pos_dev[0:1] if dyn else None)
            a = self._attention(qkv.view(B, T, 3, H, hd), T, i, kmask, pos0, cache, dyn, pos_dev, scale)
            if decode:
                thin(a.view(B * T, E), wo, ops.THIN_RES, residual=x, out=x, sumsq_out=ss_attn)
                g = thin(x, wgu, ops.THIN_SWIGLU, rms_from=(ss_attn, eps))
                thin(g, wd, ops.THIN_RES, residual=x, out=x, sumsq_out=ss_mlp)
            else:
                ops.linear_e4m3(*ops.quantize_rows_e4m3(a.view(B * T, E)), wo, residual=x, out=x, sumsq_out=ss_attn)
                g = ops.linear_e4m3(*ops.quantize_rows_e4m3(x, wgu.gain), wgu, epi=ops.EPI_SWIGLU, rms_from=(ss_attn, eps))
                ops.linear_e4m3(*ops.quantize_rows_e4m3(g), wd, residual=x, out=x, sumsq_out=ss_mlp)
        self._last_ss = None if decode else ss_mlp
        return x

    def _lm_head(self, x: torch.Tensor, rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        ops.STREAMK = self._streamk_ws(x.device)
        try:
            return self._lm_head_impl(x, rows)
        finally:
            ops.STREAMK = None

    def _lm_head_impl(self, x: torch.Tensor, rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        """final RMSNorm (as the row scale of the GEMM) + lm_head on the rows of x (reference modeling.py:508, 597)."""
        llm = self.m.llm
        gn = llm.model.norm.weight
        wl = self.derived("llm.lm_head_g", lora.weight_params(llm.lm_head) + [gn],
                          lambda: (lora.merged_weight(llm.lm_head) * gn.detach().float()[None, :]).to(ADT()).contiguous())
        ops.TAG = "lm_head"
        ss, self._last_ss = getattr(self, "_last_ss", None), None
        if rows is None and x.shape[0] > 64 and ss is not None and ss.shape[0] == x.shape[0]:
            return ops.linear(x, wl, rms_from=(ss, llm.config.rms_norm_eps))  # statistics left by the last down_proj
        rstd = ops.rms_rstd(x, llm.config.rms_norm_eps)
        if rows is not None:  # strided row subset (last position of every sample)
            x, rstd = rows, rstd.view(rows.shape[0], -1)[:, -1].contiguous()
        if x.shape[0] <= 64:
            return ops.linear_thin(x, wl, row_scale=rstd)
        return ops.linear(x, wl, row_scale=rstd)

    def llama_forward(self, embeds: torch.Tensor, attention_mask: Optional[torch.Tensor]) -> torch.Tensor:
        """Vendored LlamaModel + lm_head of the reference (modeling.py:397-522, 597) -> bf16 logits (B, T, V).

        RMSNorm rides the consuming GEMM as a per-row scale (gain folded into the weights), RoPE is applied in the QKV
        GEMM epilogue, SwiGLU in the gate/up GEMM epilogue, both residual adds in the o_proj / down_proj epilogues
        (in place on the residual stream)."""
        ops.TAG = "llama"
        self.set_format()
        B, T, E = embeds.shape
        dev = embeds.device
        x = embeds.reshape(B * T, E)
        if not x.is_contiguous():
            x = x.contiguous()
        kmask = None
        if attention_mask is not None:
            kmask = attention_mask.to(device=dev, dtype=torch.int32).contiguous()
        x = self._llama_layers(x, B, T, kmask)
        logits = self._lm_head(x)
        return logits.view(B, T, logits.shape[-1])

    # ------------------------------------------------------------------------------------------------ decoding
    def generate(self, inputs: dict, max_new_tokens: int = 128, eos_token_id: int = 2, pad_token_id: int = 32006, *,
                 do_sample: bool = False, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0,
                 repetition_penalty: float = 1.0, seed: Optional[int] = None):
        """The `inference` branch of MM_LLMs.forward (reference modeling.py:954-960):
        `llm.generate(inputs_embeds=..., max_new_tokens=128, eos_token_id=2, bos_token_id=1, pad_token_id=32006)` —
        HF generate with one beam on the multimodal prefix: greedy search, or multinomial sampling (do_sample) after
        HF's temperature / top-k (0 = off) / top-p (1.0 = off) warpers; a repetition penalty over the generated tokens
        applies in both modes.  As in the reference, NO attention mask is handed to generate (padding positions are
        attended) and only the new tokens are returned.  Prefill runs the normal forward kernels while filling a
        per-layer KV cache; every decode step is one pass of M = B GEMMs (weight-streaming bound) and a Tq = 1
        attention over the cache.  `seed` (64-bit) fixes the draws; when None it is drawn from torch's default CPU
        generator, so torch.manual_seed makes a call reproducible."""
        do_sample = bool(do_sample)
        sampler = do_sample or float(repetition_penalty) != 1.0
        if not float(repetition_penalty) > 0.0:
            raise ValueError(f"macaw_b200: repetition_penalty must be > 0, got {repetition_penalty}")
        if do_sample and not (float(temperature) > 0.0 and int(top_k) >= 0 and 0.0 <= float(top_p) <= 1.0):
            raise ValueError(f"macaw_b200: sampling needs temperature > 0, top_k >= 0 and 0 <= top_p <= 1; got "
                             f"temperature={temperature}, top_k={top_k}, top_p={top_p}")
        if do_sample and seed is None:
            lo, hi = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64).tolist()
            seed = lo | (hi << 32)
        with torch.no_grad():
            embeds, _, _ = self.prepare_inputs({k: v for k, v in inputs.items() if k not in ("labels", "attention_mask")})
            ops.TAG = "llama"
            B, T, E = embeds.shape
            dev = embeds.device
            table = self.w(self.m.llm.model.embed_tokens.weight, "llm.embed")
            n_layers = len(self.m.llm.model.layers)
            # KV buffers, step state and the captured decode graph are kept ACROSS generate() calls (keyed by batch and
            # capacity, dropped when any parameter changes): a call re-uses them instead of re-allocating 2*E*t_max*B bytes
            # per layer and re-capturing ~350 launches.  Stale rows beyond the current length are finite and masked by the
            # device-side key count, so the caches are not re-zeroed.
            t_max = _round_up(T + max_new_tokens, 64)
            stamp = self._stamp(*self.m.llm.parameters())
            kv_cls = KVCacheInt8 if self.kv_int8 else KVCache
            key = (B, t_max, str(dev), kv_cls.__name__)
            st = self._decode.get(key)
            if st is None or st["stamp"] != stamp:
                st = dict(stamp=stamp, graphs={},
                          cache=kv_cls.allocate(B, t_max, n_layers, E, dev),
                          finished=torch.zeros((B,), device=dev, dtype=torch.bool),
                          pos_dev=torch.zeros((2,), device=dev, dtype=torch.int32),
                          tok_in=torch.zeros((B,), device=dev, dtype=torch.int64))
                self._decode[key] = st
            cache, finished, pos_dev, tok_in = st["cache"], st["finished"], st["pos_dev"], st["tok_in"]
            x = embeds.reshape(B * T, E).contiguous()
            x = self._llama_layers(x, B, T, None, 0, cache, t_max)
            logits = self._lm_head(x, rows=x.view(B, T, E)[:, -1, :])
            out = torch.full((B, max_new_tokens), pad_token_id, device=dev, dtype=torch.int64)
            finished.zero_()
            pad = torch.full((B,), pad_token_id, device=dev, dtype=torch.int64)
            graph_key = (int(eos_token_id), int(pad_token_id))
            if sampler:
                # The generated-token bitmap starts empty (HF's input_ids are empty when generate gets only
                # inputs_embeds); seed and step live on the device, so the captured decode graph draws fresh numbers.
                V = logits.shape[1]
                if "seen" not in st:
                    st["seen"] = torch.zeros((B, (V + 31) // 32), device=dev, dtype=torch.int32)
                    st["seed_dev"] = torch.zeros((1,), device=dev, dtype=torch.int64)
                    st["step_dev"] = torch.zeros((1,), device=dev, dtype=torch.int32)
                seen, seed_dev, step_dev = st["seen"], st["seed_dev"], st["step_dev"]
                seen.zero_()
                step_dev.zero_()
                s64 = (int(seed or 0) & (2 ** 64 - 1))
                seed_dev.fill_(s64 - 2 ** 64 if s64 >= 2 ** 63 else s64)
                cfg = dict(do_sample=do_sample, repetition_penalty=float(repetition_penalty),
                           temperature=float(temperature), top_k=int(top_k), top_p=float(top_p))
                graph_key += tuple(cfg.values())

                def pick(lg):
                    t = ops.sample_rows(lg, seen, seed_dev=seed_dev, step_dev=step_dev, **cfg)
                    step_dev.add_(1)
                    return t
            else:
                pick = ops.argmax_rows
            tok = pick(logits)
            out[:, 0] = tok
            finished |= tok == eos_token_id
            n = 1
            if max_new_tokens > 1 and not bool(finished.all()):
                # One decode step = ~10 launches per layer: host-bound when launched one by one, so the step is captured
                # ONCE in a CUDA graph whose kernels read position / cache slot / key count from `pos_dev`.
                pos_dev.copy_(torch.tensor([T, T + 1], dtype=torch.int32), non_blocking=True)
                tok_in.copy_(tok)
                eos_t, pad_t = int(eos_token_id), pad

                def decode_step():
                    x1 = ops.embed_gather(table, tok_in)  # ids beyond the table (pad of finished rows) are clamped
                    x1 = self._llama_layers(x1, B, 1, None, 1, cache, t_max, pos_dev)
                    nxt = pick(self._lm_head(x1))
                    nxt = torch.where(finished, pad_t, nxt)  # HF: finished rows emit pad
                    finished.logical_or_(nxt == eos_t)
                    tok_in.copy_(nxt)
                    pos_dev.add_(1)

                # one captured decode step per (eos, pad[, sampling configuration]): alternating greedy and sampled
                # calls replay their own graphs
                graph = st["graphs"].get(graph_key, (None,))[0]
                if graph is None:
                    decode_step()  # eager first step: fills weight caches / function attributes, and is a real step
                    out[:, 1] = tok_in
                    n = 2
                while n < max_new_tokens:
                    if n % 8 == 2 and bool(finished.all()):  # host check every 8 steps (finished rows only emit pad)
                        break
                    if graph is None:
                        graph = torch.cuda.CUDAGraph()
                        prof, ops.PROFILE = ops.PROFILE, None
                        try:
                            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                                decode_step()
                        finally:
                            ops.PROFILE = prof
                        st["graphs"][graph_key] = (graph, pad_t)  # the captured pad tensor lives with its graph
                    graph.replay()
                    out[:, n] = tok_in
                    n += 1
                # trim trailing all-pad columns produced between two host checks
                alive = (out[:, :n] != pad_token_id).any(dim=0)
                n = int(alive.nonzero().max().item()) + 1 if bool(alive.any()) else 1
        return out[:, :n]

    # ------------------------------------------------------------------------------------------------ whole forward
    def _forward_eager(self, inputs: dict):
        with torch.no_grad():
            embeds, mask, labels = self.prepare_inputs(inputs)
            logits = self.llama_forward(embeds, mask)
            loss = ops.ce_loss(logits, labels) if labels is not None else None
        return loss, logits, embeds, mask, labels

    def forward(self, inputs: dict):
        """MM_LLMs.forward (reference modeling.py:941-963), prefill branch -> (loss | None, logits (B, T, V) bf16, ...)."""
        if self._graphs_on:
            return self._forward_graphed(inputs)
        return self._forward_eager(inputs)

    # ---- CUDA-graph replay of the whole forward (opt-in) -----------------------------------------------------
    def enable_cuda_graphs(self, flag: bool = True) -> None:
        """Capture the ~480 kernel launches of one forward into a CUDA graph per input signature and replay it.

        Removes per-launch host overhead (matters at small per-GPU batch).  Opt-in because the returned tensors are
        STATIC buffers: a later call with the same input signature overwrites them.  Graphs are re-captured when
        any parameter's version changes."""
        self._graphs_on = bool(flag)
        if not flag:
            self._graphs.clear()

    def enable_int8_kv_cache(self, flag: bool = True) -> None:
        """Keep generate()'s KV cache in int8 (KVCacheInt8: one fp32 scale per token and head for keys and for values),
        about half the bytes of the 16-bit cache.  The prefill's attention still reads its fresh 16-bit q / k / v, so the
        first generated token is the 16-bit cache's; decode steps attend over the dequantized cache.  The decode state
        is dropped, so the other format's buffers are freed.  The eval forward and the training step are unaffected."""
        self.kv_int8 = bool(flag)
        self._decode.clear()

    _TENSOR_KEYS = ("images", "audios", "videos", "input_ids", "attention_mask", "labels", "image_starts", "image_ends",
                    "audio_starts", "audio_ends", "video_starts", "video_ends")

    def _forward_graphed(self, inputs: dict):
        self.set_format()
        dev = self.w(self.m.llm.model.embed_tokens.weight, "llm.embed").device
        # graphs bake parameter ADDRESSES in: any replaced Parameter (resize_token_embeddings), `.data` swap (model.to)
        # or in-place update (optimizer step) must drop them — same key the derived-weight cache uses
        stamp = self._stamp(*self.m.parameters())
        present = tuple((k, tuple(inputs[k].shape)) for k in self._TENSOR_KEYS
                        if isinstance(inputs.get(k), torch.Tensor))
        key = (present, str(dev))
        ent = self._graphs.get(key)
        if ent is not None and ent[3] != stamp:
            ent = None
        if ent is None:
            static_in = {k: v for k, v in inputs.items() if not isinstance(v, torch.Tensor)}
            for k, _ in present:
                v = inputs[k]
                dt = ADT() if v.is_floating_point() else v.dtype
                static_in[k] = torch.empty(v.shape, device=dev, dtype=dt)
                static_in[k].copy_(v, non_blocking=True)
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                for _ in range(2):  # populate weight caches / function attributes before capture
                    self._forward_eager(static_in)
            cur.wait_stream(side)
            torch.cuda.synchronize(dev)
            g = torch.cuda.CUDAGraph()
            prof, ops.PROFILE = ops.PROFILE, None  # event timing cannot live inside a capture
            try:
                with torch.cuda.graph(g, capture_error_mode="thread_local"):
                    out = self._forward_eager(static_in)
            finally:
                ops.PROFILE = prof
            ent = (g, static_in, out, stamp)
            self._graphs[key] = ent
        else:
            static_in = ent[1]
            for k, _ in present:
                v = inputs[k]
                if v.data_ptr() != static_in[k].data_ptr():
                    static_in[k].copy_(v, non_blocking=True)
        ent[0].replay()
        return ent[2]
