"""Device-side input pipeline (SURVEY.md §8f rank 3): `LLMTrainer.get_self_inputs` of the reference
(/root/reference/llm_trainer.py:306-381) with the per-sample pixel / audio arithmetic moved onto the GPU.

  reference (host, inside every step)                        here
  ------------------------------------------------------     ------------------------------------------------------------
  PIL decode -> Resize(224, BICUBIC) -> CenterCrop(224) ->    decoded 8-bit RGB pixels are uploaded once; mm_image_preprocess
  ToTensor -> Normalize (llm_trainer.py:151-158, 318-320)     does Pillow's antialiased two-pass bicubic resize (bit-exact
                                                              8-bit result), the crop, /255 and the CLIP mean / std
  whisper.load_audio -> pad_or_trim -> log_mel_spectrogram    decoded 16 kHz PCM is uploaded; mm_log_mel evaluates the
  (llm_trainer.py:338-345)                                    STFT / mel / log / clamp pipeline (30 s -> 80 x 3000)
  .half(), .to(device)  (:366-379)                            outputs are produced on the device in the model dtype

JPEG files (images and pre-extracted video frames, `'{}{}.mp4_{}.jpg'` in the reference) are decoded on the device too,
bit-exactly as Pillow decodes them (jpeg.py, csrc/jpeg.cu): `image()`, `images()`, `videos()` and `get_self_inputs()` take
JPEG bytes or file paths next to decoded arrays, and every JPEG of one call goes through one batched decode.  Files the
device decoder refuses (progressive, CMYK, ...) raise; decode those on the host and pass the array.  Audio-container
decoding stays on the host (ffmpeg in the reference): this module takes decoded PCM.
The coefficient tables of the resize are built here with Pillow's exact double-precision arithmetic (Resample.c:
precompute_coeffs + normalize_coeffs_8bpc) and cached per source size; the windowed DFT basis and the mel filter bank
(librosa's Slaney filters, as shipped in whisper/assets/mel_filters.npz) are built once per device.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, jpeg, ops, wire

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)   # llm_trainer.py:157
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
N_SAMPLES, N_FFT, HOP, N_MELS, N_FRAMES, SAMPLE_RATE = 480000, 400, 160, 80, 3000, 16000
PRECISION_BITS = 32 - 8 - 2


# ---------------------------------------------------------------------------------------------------- Pillow resampling
def _bicubic(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def pillow_coeffs(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray, int]:
    """Pillow's precompute_coeffs (bicubic, support 2) + normalize_coeffs_8bpc for a whole-axis resize in_size -> out_size:
    (bounds int32 [out][2] = (first source index, tap count), coefficients int32 [out][ksize], ksize)."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    kk = np.zeros((out_size, ksize), dtype=np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        xmax -= xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x in range(xmax):
            v = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, kk, ksize


def resize_geometry(h: int, w: int, size: int = 224) -> dict:
    """torchvision Resize(size) (shorter side -> size, longer = int(size * long / short)) followed by CenterCrop(size)
    (offsets int(round((dim - size) / 2.0)), python rounding)."""
    if w <= h:
        new_w, new_h = size, int(size * h / w)
    else:
        new_h, new_w = size, int(size * w / h)
    top = int(round((new_h - size) / 2.0))
    left = int(round((new_w - size) / 2.0))
    return dict(new_h=new_h, new_w=new_w, top=top, left=left)


class DeviceInputPipeline:
    """Builds the `inputs` dict of llm_trainer.py:363-381 from decoded media with the arithmetic on the GPU."""

    def __init__(self, device="cuda", dtype=torch.bfloat16, image_size: int = 224, n_frames: int = 6):
        self.dev = torch.device(device)
        self.dtype = dtype
        self.size = image_size
        self.n_frames = n_frames
        self._tables: Dict[Tuple[int, int], dict] = {}
        self._audio = None

    # ---- images
    def _image_tables(self, h: int, w: int) -> dict:
        t = self._tables.get((h, w))
        if t is None:
            g = resize_geometry(h, w, self.size)
            bh, kh, ksh = pillow_coeffs(w, g["new_w"])
            bv, kv, ksv = pillow_coeffs(h, g["new_h"])
            bh, kh = bh[g["left"]: g["left"] + self.size], kh[g["left"]: g["left"] + self.size]
            bv, kv = bv[g["top"]: g["top"] + self.size], kv[g["top"]: g["top"] + self.size]
            row0 = int(bv[:, 0].min())
            row1 = int((bv[:, 0] + bv[:, 1]).max())
            t = dict(geom=g, ksh=ksh, ksv=ksv, row0=row0, n_rows=row1 - row0,
                     bh=torch.from_numpy(np.ascontiguousarray(bh)).to(self.dev), kh=torch.from_numpy(np.ascontiguousarray(kh)).to(self.dev),
                     bv=torch.from_numpy(np.ascontiguousarray(bv)).to(self.dev), kv=torch.from_numpy(np.ascontiguousarray(kv)).to(self.dev))
            self._tables[(h, w)] = t
        return t

    def decode_jpegs(self, items: Sequence) -> List[torch.Tensor]:
        """JPEG files (`bytes`, or `str` / `os.PathLike` paths) -> uint8 (H, W, 3) RGB device tensors, decoded in one batch
        on the device, bit-exact with `np.asarray(Image.open(f))` (grayscale files come back with the plane replicated).
        Raises NotImplementedError for a JPEG variant the decoder does not support, ValueError for a corrupt file."""
        return jpeg.decode(items, self.dev)

    def _decode_items(self, images: Sequence, videos: Sequence) -> Tuple[list, list]:
        """images / videos with every JPEG item replaced by its decoded array, all of them in one batched decode."""
        items = [r for r in images if jpeg.is_item(r)] + [f for fs in videos if fs is not None for f in fs if jpeg.is_item(f)]
        if not items:
            return list(images), list(videos)
        it = iter(self.decode_jpegs(items))
        images = [next(it) if jpeg.is_item(r) else r for r in images]
        videos = [fs if fs is None else [next(it) if jpeg.is_item(f) else f for f in fs] for fs in videos]
        return images, videos

    def image(self, rgb, out: Optional[torch.Tensor] = None, want_u8: bool = False, fp32: bool = False):
        """One image: uint8 (H, W, 3) RGB (host or device), or a JPEG file (bytes / path, decoded on the device) ->
        (3, size, size) in the pipeline dtype (fp32 when asked).  Returns (tensor, uint8 HWC resized+cropped image | None)."""
        if jpeg.is_item(rgb):
            rgb = self.decode_jpegs([rgb])[0]
        if rgb.dtype != torch.uint8 or rgb.dim() != 3 or rgb.shape[2] != 3:
            raise ValueError("image(): expected a uint8 (H, W, 3) RGB array (decode / convert('RGB') on the host first)")
        src = rgb.to(self.dev, non_blocking=True).contiguous()
        h, w = int(src.shape[0]), int(src.shape[1])
        t = self._image_tables(h, w)
        S = self.size
        dt = torch.float32 if fp32 else self.dtype
        if dt not in (torch.float32, torch.bfloat16):
            raise TypeError("image(): output dtype must be bf16 or fp32")
        if out is None:
            out = torch.empty((3, S, S), device=self.dev, dtype=dt)
        assert out.is_contiguous() and out.shape == (3, S, S) and out.dtype == dt
        tmp = torch.empty((t["n_rows"], S, 3), device=self.dev, dtype=torch.uint8)
        u8 = torch.empty((S, S, 3), device=self.dev, dtype=torch.uint8) if want_u8 else None
        a = _lib.ImageArgs(src.data_ptr(), src.stride(0), t["row0"], t["n_rows"], S, S, t["bh"].data_ptr(), t["kh"].data_ptr(),
                           t["ksh"], t["bv"].data_ptr(), t["kv"].data_ptr(), t["ksv"], (C.c_float * 3)(*CLIP_MEAN),
                           (C.c_float * 3)(*CLIP_STD), tmp.data_ptr(), out.data_ptr(), int(dt == torch.float32),
                           None if u8 is None else u8.data_ptr())
        with torch.cuda.device(self.dev):
            ops._check(_lib.load().mm_image_preprocess(C.byref(a), ops._stream()), "mm_image_preprocess")
        return out, u8

    def images(self, rgbs: Sequence[Optional[torch.Tensor]]) -> torch.Tensor:
        """A batch of images, decoded arrays or JPEG files (None = absent -> zeros, llm_trainer.py:352) -> (B, 3, size, size)."""
        rgbs, _ = self._decode_items(rgbs, [])
        out = torch.zeros((len(rgbs), 3, self.size, self.size), device=self.dev, dtype=self.dtype)
        for i, r in enumerate(rgbs):
            if r is not None:
                self.image(r, out=out[i])
        return out

    def videos(self, frames: Sequence[Optional[Sequence[torch.Tensor]]]) -> torch.Tensor:
        """Per sample a list of n_frames frames, decoded arrays or JPEG files (None = absent -> zeros, llm_trainer.py:315)
        -> (B, F, 3, S, S)."""
        _, frames = self._decode_items([], frames)
        out = torch.zeros((len(frames), self.n_frames, 3, self.size, self.size), device=self.dev, dtype=self.dtype)
        for i, fs in enumerate(frames):
            if fs is None:
                continue
            if len(fs) != self.n_frames:
                raise ValueError(f"videos(): expected {self.n_frames} frames per sample, got {len(fs)}")
            for j, r in enumerate(fs):
                self.image(r, out=out[i, j])
        return out

    # ---- audio
    def _audio_tables(self):
        if self._audio is None:
            n = np.arange(N_FFT, dtype=np.float64)
            window = 0.5 - 0.5 * np.cos(2.0 * np.pi * n / N_FFT)  # torch.hann_window(400) (periodic)
            f = np.arange(N_FFT // 2 + 1, dtype=np.float64)
            ang = 2.0 * np.pi * np.outer(n, f) / N_FFT            # [400][201]
            basis = np.zeros((N_FFT, 2, 208), dtype=np.float32)
            basis[:, 0, :201] = (window[:, None] * np.cos(ang)).astype(np.float32)
            basis[:, 1, :201] = (-window[:, None] * np.sin(ang)).astype(np.float32)
            mel = mel_filters().astype(np.float32)                # [80][201]
            self._audio = (torch.from_numpy(basis).to(self.dev), torch.from_numpy(np.ascontiguousarray(mel)).to(self.dev))
        return self._audio

    def log_mel(self, pcm: torch.Tensor, out: Optional[torch.Tensor] = None, fp32: bool = False) -> torch.Tensor:
        """One clip: fp32 PCM at 16 kHz (any length; padded / trimmed to 30 s) -> (80, 3000)."""
        if pcm.dim() != 1 or not pcm.is_floating_point():
            raise ValueError("log_mel(): expected a 1-D floating point waveform at 16 kHz")
        x = pcm.to(self.dev, torch.float32, non_blocking=True).contiguous()
        basis, mel = self._audio_tables()
        dt = torch.float32 if fp32 else self.dtype
        if out is None:
            out = torch.empty((N_MELS, N_FRAMES), device=self.dev, dtype=dt)
        assert out.is_contiguous() and out.shape == (N_MELS, N_FRAMES) and out.dtype == dt
        logspec = torch.empty((N_MELS, N_FRAMES), device=self.dev, dtype=torch.float32)
        mx = torch.empty((1,), device=self.dev, dtype=torch.int32)
        with torch.cuda.device(self.dev):
            ops._check(_lib.load().mm_log_mel(x.data_ptr(), min(int(x.numel()), N_SAMPLES), basis.data_ptr(), mel.data_ptr(),
                                              logspec.data_ptr(), mx.data_ptr(), out.data_ptr(), int(dt == torch.float32),
                                              ops._stream()), "mm_log_mel")
        return out

    def audios(self, pcms: Sequence[Optional[torch.Tensor]]) -> torch.Tensor:
        """A batch of clips (None = absent -> zeros, llm_trainer.py:332) -> (B, 80, 3000)."""
        out = torch.zeros((len(pcms), N_MELS, N_FRAMES), device=self.dev, dtype=self.dtype)
        for i, p in enumerate(pcms):
            if p is not None:
                self.log_mel(p, out=out[i])
        return out

    # ---- the reference's get_self_inputs
    def get_self_inputs(self, batch: Dict[str, torch.Tensor], images: Sequence[Optional[torch.Tensor]],
                        audios: Sequence[Optional[torch.Tensor]], videos: Sequence[Optional[Sequence[torch.Tensor]]]) -> dict:
        """llm_trainer.py:306-381 with media instead of file names: images and video frames as decoded arrays or JPEG files
        (all JPEGs of the call decoded in one batch), audio as decoded PCM; `batch` carries input_ids / attention_mask /
        labels (wire.collate); returns {'inputs': {...}} exactly like the reference."""
        dev = self.dev
        images, videos = self._decode_items(images, videos)
        d = {
            "videos": self.videos(videos), "audios": self.audios(audios), "images": self.images(images),
            "input_ids": batch["input_ids"].to(dev), "attention_mask": batch["attention_mask"].to(dev),
            "labels": batch["labels"].to(dev) if batch.get("labels") is not None else None,
        }
        B = d["input_ids"].shape[0]
        for name in ("image", "audio", "video"):
            d[f"{name}_starts"] = torch.full((B,), wire.SPECIAL_TOKENS[f"<{name}>"], dtype=torch.int32, device=dev)
            d[f"{name}_ends"] = torch.full((B,), wire.SPECIAL_TOKENS[f"</{name}>"], dtype=torch.int32, device=dev)
        return {"inputs": d}


# ---------------------------------------------------------------------------------------------------- mel filter bank
def mel_filters(sr: int = SAMPLE_RATE, n_fft: int = N_FFT, n_mels: int = N_MELS) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels) (Slaney mel scale, Slaney area normalisation, fmin 0, fmax sr/2): the
    filter bank whisper ships as assets/mel_filters.npz and log_mel_spectrogram multiplies by.  -> [n_mels][n_fft//2+1]."""
    def hz_to_mel(f):
        f = np.asarray(f, dtype=np.float64)
        f_sp = 200.0 / 3
        mels = f / f_sp
        min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
        return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, mels)

    def mel_to_hz(m):
        m = np.asarray(m, dtype=np.float64)
        f_sp = 200.0 / 3
        min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
        return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)

    fftfreqs = np.linspace(0, sr / 2.0, n_fft // 2 + 1)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(sr / 2.0), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    weights = np.zeros((n_mels, n_fft // 2 + 1), dtype=np.float64)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2: n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, None]
    return weights.astype(np.float32)
