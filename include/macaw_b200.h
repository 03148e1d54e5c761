/*
 * macaw_b200.h — C ABI of libmacaw_b200.so, the sm_90a kernel library behind the MM_LLMs forward hot path.
 *
 * The reference (lyuchenyang/Macaw-LLM) has no FFI layer of its own: its hot path is Python calling
 * torch / transformers modules (SURVEY.md §8b).  Each entry point below therefore cites the reference
 * call site(s) whose arithmetic it replaces; the Python host code in macaw-llm_b200/ binds them with
 * ctypes (INTEGRATION.md shows the stub a maintainer of the reference would add).
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on error; mm_last_error() returns a message for the
 *     calling thread.  No exceptions cross this boundary and nothing here calls cudaMalloc.  mm_host_alloc /
 *     mm_host_free (page-locked host memory for optimizer state) are the library's ONLY allocating entries; they are
 *     called when an optimizer is set up and torn down, never inside a training step.
 *   - all pointers are DEVICE pointers owned by the caller (torch's caching allocator in practice), or device aliases of
 *     mm_host_alloc memory where a function says so.
 *   - `stream` is a cudaStream_t passed as void*; all calls are asynchronous and never synchronise.
 *   - "bf16" means 16-bit bfloat16 storage, row-major unless a leading dimension says otherwise; all
 *     accumulation is fp32.
 */
#ifndef MACAW_B200_H_
#define MACAW_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------ meta */
const char* mm_last_error(void);
int32_t mm_abi_version(void);
/* Content hash of the kernel sources + this header the library was built from (the loader compares it with the sources
 * on disk and rebuilds on mismatch, so a stale library never meets a newer struct layout). */
const char* mm_build_hash(void);
/* Number of kernel launches issued through this library by the calling process since the last reset. */
int64_t mm_launch_count(void);
void mm_launch_count_reset(void);
/* 16-bit storage format of activations and parameters for the CALLING THREAD: 0 = bf16 (default), 1 = fp16 (IEEE half).
 * Wherever this header says "bf16" for an activation / parameter tensor, the tensor is fp16 while the format is 1.  The
 * reference itself trains and runs in fp16 (train.sh:36 `--fp16 True`, llm_trainer.py:366-368 `.half()`); an fp16 model is
 * computed in fp16 (11-bit significands: storage rounding 8x smaller than bf16), a bf16 model in bf16.  mm_gemm_fwd and
 * mm_align_fwd take their operand formats explicitly; they use this flag for the epilogue's bias / residual tensors. */
void mm_set_act_format(int32_t f16);
int32_t mm_get_act_format(void);

/* ------------------------------------------------------------------------------------------------ GEMM
 * C[b] = epilogue( alpha * A[b] (M x K, K contiguous) * B[b]^T ) for b in [0, batch).
 * Replaces every nn.Linear / Conv-as-matmul / bmm on the path:
 *   LLaMA q/k/v/o/gate/up/down/lm_head   modeling.py:134-140, 159-162, 179-181, 226, 597
 *   alignment MHA in/out projections      modeling.py:986-987, 1007-1008, 1025-1026 -> torch F.multi_head_attention_forward
 *   Conv1d down-samplers, Linear C->E     modeling.py:982-984, 999-1001, 1022-1024
 *   CLIP / Whisper encoder linears, convs  modeling.py:1073, 1082, 1092 -> transformers modeling_clip / modeling_whisper
 * Implementation: persistent, warp-specialised TMA -> wgmma kernel (register accumulators, two consumer warpgroups).
 */
enum {
  MM_ACT_NONE = 0,
  MM_ACT_GELU = 1,        /* exact erf GELU (Whisper) */
  MM_ACT_QUICK_GELU = 2,  /* x * sigmoid(1.702 x) (CLIP) */
  MM_ACT_SILU = 3
};
enum {
  MM_EPI_STD = 0,    /* bias / activation / residual */
  MM_EPI_SWIGLU = 1, /* B rows interleaved [32 gate | 32 up]; C[:, j] = silu(gate_j) * up_j, N_out = N/2 */
  MM_EPI_ROPE = 2    /* rotate-half RoPE (head_dim 128) on columns < rope_cols, pos = row % rope_T */
};

typedef struct mm_gemm_args {
  /* problem: batch (inner) x batch2 (outer, 0 or 1 = none) independent products */
  int32_t M, N, K, batch, batch2;
  /* A: bf16 [batch][M][K], row stride lda (elements), batch stride a_bs (elements; rows may overlap) */
  const void* A;
  int64_t lda, a_bs, a_bs2;
  /* B: bf16.  b_mn_major == 0: [batch][N][K] (K contiguous, i.e. an nn.Linear weight), row stride ldb.
   *           b_mn_major == 1: [batch][K][N] (N contiguous), row stride ldb.  b_bs == 0 shares B across batch. */
  const void* B;
  int64_t ldb, b_bs, b_bs2;
  int32_t b_mn_major;
  /* C: bf16 (c_fp32 == 0) or fp32 (c_fp32 == 1) [batch][M][N_out], row stride ldc */
  void* C;
  int64_t ldc, c_bs, c_bs2;
  int32_t c_fp32;
  /* epilogue */
  int32_t epi;            /* MM_EPI_* */
  int32_t act;            /* MM_ACT_* (MM_EPI_STD only) */
  float alpha;
  const void* bias;       /* bf16 [N] or NULL; bias_bs = per-batch stride in elements */
  int64_t bias_bs;
  const float* row_scale; /* fp32 [batch2*batch*M] or NULL: multiplies row m of the product before bias */
  const void* residual;   /* bf16, added after activation; row index = m % res_row_mod if res_row_mod > 0 */
  int64_t ldr, r_bs, r_bs2;
  int32_t res_row_mod;
  const float* rope_cos;  /* fp32 [rope_T][64] */
  const float* rope_sin;
  int32_t rope_T, rope_cols;
  const int32_t* rope_pos; /* NULL, or device int added to every row's position (decode steps replayed from a CUDA graph) */
  int32_t c_trans; /* 1: C and residual are addressed transposed (C[n][m], row stride ldc), bias is indexed by m, row_scale by n:
                      lets a caller swap the operands (A = weight rows, B = a handful of activation rows) so that thin
                      decode GEMMs fill the 128-row MMA tile with weights (standard epilogue, batch == 1) */
  /* 16-bit operand formats: 0 = bf16 (default), 1 = fp16 (IEEE half).  A and B must agree: wgmma takes one input type
   * for both operands.
   * The alignment chain runs in fp16 (11-bit significand: one stored stage costs 1.4e-4 norm-wise instead of bf16's
   * 1.1e-3) against fp16 COPIES of its weights and of the embedding table (exact conversions of the bf16 values). */
  int32_t a_fp16, b_fp16;
  int32_t c_fp16; /* 1: C is fp16 (c_fp32 must be 0) */
  /* MM_EPI_STD only: out += bias_rs[b*M + m] * bias[n] (when bias_rs != NULL the bias term is scaled per row) and
   * out += bias2_rs[b*M + m] * bias2[n].  Value-side bias terms of the absorbed alignment attention
   * (functional.py:6531-6537: b_v rides on every real key, bias_v on the appended key). bias2 shares bias_bs. */
  const float* bias_rs;
  const void* bias2;
  const float* bias2_rs;
  /* 1: A is given as [batch][K][M] (M contiguous, row stride lda) — the transpose of a row-major activation.  With
   * b_mn_major this is the weight-gradient product dW[n][k] = sum_m dY[m][n] X[m][k] on the tensors as stored
   * (reference: autograd of every nn.Linear on the path; llm_trainer.py:184-188 -> loss.backward()). */
  int32_t a_mn_major;
  /* RMSNorm statistics without a separate pass over the residual stream (LlamaRMSNorm modeling.py:311-319):
   * sumsq_out (MM_EPI_STD, 16-bit C): fp32 [M][ceil(N/32)] — the epilogue that WRITES the new residual stream also writes,
   * per row and 32-column chunk, the sum of squares of the values as stored.  rs_sumsq (any epilogue): fp32 [M][rs_parts] —
   * the GEMM that CONSUMES the stream derives its per-row scale rsqrt(sum / K + rs_eps) from those partials (fixed
   * summation order: deterministic) instead of reading `row_scale`. */
  float* sumsq_out;
  const float* rs_sumsq;
  int32_t rs_parts;
  float rs_eps;
  /* Stream-K tail (optional; null = plain data-parallel tiles).  When the tile count leaves a partial last wave
   * (e.g. 288 tiles on 132 SMs), the tail's k-blocks are divided evenly over ALL CTAs; partial fp32 accumulators pass
   * through this workspace: 8192 bytes of flags (zero before the first use, self-resetting afterwards) followed by one
   * 128 x 128 fp32 slot per SM — mm_gemm_streamk_workspace_bytes().  One workspace must not be used by GEMMs running
   * CONCURRENTLY on different streams.  Ignored for launches without one full wave of tiles (the tail pieces run first
   * and hide their hand-over behind the full tiles). */
  void* sk_workspace;
  int64_t sk_workspace_bytes;
} mm_gemm_args;

int32_t mm_gemm_fwd(const mm_gemm_args* args, void* stream);
/* The schedule mm_gemm_fwd would use for `args` on the current device (132 SMs when no device is visible), without
 * touching memory or launching: the host-side decisions — tile width from the cost model, rasterisation group,
 * stream-K tail, kernel variant and launch shape — are a pure function of the shapes, strides, alignments and flags.
 * Operand pointers are only checked for null / alignment, never dereferenced.  Host logic made testable without a GPU
 * (tests/test_gemm_plan.py) and printable per BASELINE shape (tools/gemm_plan.py).
 * m_tiles, n_tiles, units and waves describe the 128 x block_n tile grid whichever kernel runs it; kernel, threads,
 * grid and smem_bytes describe the launch itself (a TILE_PAIRS CTA takes two N-neighbouring tiles at a time). */
enum {
  MM_GEMM_KERNEL_CONSUMER_EPILOGUE = 0,  /* 288 threads: the consumer warpgroups run each tile's epilogue */
  MM_GEMM_KERNEL_EPILOGUE_WARPGROUP = 1, /* 512 threads: a dedicated epilogue warpgroup (mm_gemm_overlap_mode 1, 2) */
  MM_GEMM_KERNEL_TILE_PAIRS = 2          /* 384 threads: two 128-wide tiles per 128 x 256 main loop (mode 2) */
};
typedef struct mm_gemm_schedule {
  int32_t block_n;             /* tile = 128 x block_n x 64 */
  int32_t kernel;              /* MM_GEMM_KERNEL_*: the kernel variant launched */
  int32_t m_tiles, n_tiles, k_blocks;
  int64_t units;               /* work units over all batches: tiles */
  int32_t workers;             /* units in flight: SMs */
  int32_t grid;                /* CTAs launched (persistent: <= SM count) */
  int32_t threads;             /* threads per CTA */
  int32_t waves;               /* ceil(units / workers) */
  int32_t group_m;             /* rasterisation: M units per L2 group */
  int32_t streamk_tiles;       /* tiles of the partial last wave shared over all CTAs (0 = plain tiles) */
  int32_t smem_bytes;          /* dynamic shared memory per CTA */
  int32_t vectorised_epilogue; /* 1 = 128-bit epilogue accesses (all alignments hold) */
} mm_gemm_schedule;
int32_t mm_gemm_plan(const mm_gemm_args* args, mm_gemm_schedule* plan);
/* Stream-K policy of the process: 0 never, 1 when the saved MMA time exceeds the hand-over cost (default; environment
 * MACAW_B200_GEMM_STREAMK), 2 whenever the schedule allows (tests).  mode < 0 only queries.  Returns the previous mode. */
int32_t mm_gemm_streamk_mode(int32_t mode);
/* Epilogue-overlap policy of the process: 0 the consumer warpgroups run each tile's epilogue themselves, 1 a dedicated
 * epilogue warpgroup runs it while they start the next tile, 2 as 1 and launches whose 128-wide N tiles pair up walk
 * them two at a time under one 128 x 256 main loop (default; environment MACAW_B200_GEMM_OVERLAP).  Outputs are
 * bit-identical in all modes.  mode < 0 only queries.  Returns the previous mode. */
int32_t mm_gemm_overlap_mode(int32_t mode);
/* bytes of mm_gemm_args.sk_workspace on the current device */
int64_t mm_gemm_streamk_workspace_bytes(void);

/* Sum fp32 partials [splits][M][N] (+ bf16 bias[N]) -> bf16 (or fp16 when out_fp16 != 0) [M][N] (row stride ldo).
 * Split-K tail of the Conv1d down-samplers (modeling.py:982, 999, 1022). */
int32_t mm_splitk_reduce(const float* partial, int32_t splits, int32_t M, int32_t N, const void* bias, void* out,
                         int64_t ldo, int32_t out_fp16, void* stream);

/* ------------------------------------------------------------------------------------------------ attention
 * out[b,t,h,:] = softmax(scale * q k^T + mask) v, flash-style (no T x T tensor in HBM).
 * Replaces: LlamaAttention.forward modeling.py:197-215 (causal + key padding), CLIP / Whisper encoder
 * self-attention (transformers modeling_clip.py / modeling_whisper.py eager attention), and
 * video_long_self_attention modeling.py:1078 (two synthetic keys are materialised by the caller).
 * q/k/v/out: bf16 with element strides (batch, token, head); head_dim contiguous, head_dim in {64, 96, 128}.
 * key_mask: int32 [B][Tk] (1 = attend, 0 = masked) or NULL.  causal: key j visible to query i iff j <= i + (Tk - Tq).
 * scale > 0.
 */
typedef struct mm_attn_args {
  const void *q, *k, *v;
  void* out;
  int32_t B, H, Tq, Tk, head_dim;
  int64_t q_bs, q_ts, q_hs;
  int64_t k_bs, k_ts, k_hs;
  int64_t v_bs, v_ts, v_hs;
  int64_t o_bs, o_ts, o_hs;
  const int32_t* key_mask;
  int32_t causal;
  float scale;
  const int32_t* tk_dev; /* NULL, or device int holding the number of valid keys (<= Tk, which then is the capacity of
                            k / v): lets one captured launch serve a growing KV cache */
} mm_attn_args;
int32_t mm_attn_fwd(const mm_attn_args* args, void* stream);

/* ------------------------------------------------------------------------------------------------ norms
 * LlamaRMSNorm modeling.py:311-319 (fp32 variance);  y = x * rsqrt(mean(x^2) + eps) * w.  x, y bf16 [rows][cols]. */
int32_t mm_rmsnorm_fwd(const void* x, const void* w, void* y, int32_t rows, int32_t cols, float eps, void* stream);
/* rstd[r] = rsqrt(mean(x[r]^2) + eps) (fp32): the row statistic of LlamaRMSNorm.  With the gain folded into the next
 * Linear's weight (W' = W * diag(g)) the norm itself becomes the `row_scale` of that GEMM's epilogue:
 * RMSNorm(x) W^T = rstd * (x W'^T), so the normalised activations are never written to HBM. */
int32_t mm_rms_rstd(const void* x, float* rstd, int32_t rows, int32_t cols, float eps, void* stream);
/* nn.LayerNorm of the CLIP / Whisper encoders (transformers modeling_clip.py:CLIPEncoderLayer, modeling_whisper.py). */
int32_t mm_layernorm_fwd(const void* x, int64_t ldx, const void* w, const void* b, void* y, int64_t ldy, int32_t rows,
                         int32_t cols, float eps, void* stream);

/* ------------------------------------------------------------------------------------------------ gathers / layout
 * embed_tokens lookup modeling.py:971-972, 979-980, 996-997, 1019-1020: out[i,:] = table[ids[i],:] (ids int64). */
int32_t mm_embed_gather(const void* table, int32_t vocab, int32_t dim, const int64_t* ids, int64_t n_ids, void* out,
                        int64_t ldo, void* stream);
/* Splice modeling.py:989-993, 1010-1016, 1028-1034 done in one pass.
 * dst (B, T, E) bf16 with T = 1 + n_prefix + (L-1):  dst[b,0] = text[b,0]; dst[b,1+j] = prefix[b,j]; dst[b,1+n_prefix+j] = text[b,1+j].
 * Also builds the int64 mask/label prefix of modeling.py:1036-1046 (bit-exact): mask_out = [1]*n_prefix ++ mask_in,
 * labels_out = [-100]*n_prefix ++ labels_in.  mask_in/labels_in may be NULL (then the outputs are not written). */
int32_t mm_splice_prefix(const void* text, const void* prefix, void* dst, int32_t B, int32_t L, int32_t n_prefix,
                         int32_t E, const int64_t* mask_in, int64_t* mask_out, const int64_t* labels_in,
                         int64_t* labels_out, void* stream);
/* CLIP patch embedding im2col (transformers modeling_clip.py:CLIPVisionEmbeddings): images (B,3,H,W) bf16 ->
 * rows (B*gh*gw, ldo) with column order (c, py, px); columns >= 3*p*p are zero. */
int32_t mm_patchify(const void* images, int32_t B, int32_t C, int32_t H, int32_t W, int32_t patch, void* out,
                    int64_t ldo, void* stream);
/* (B, C, T) -> (B, T + 2*pad, C) with zero pad rows (Whisper conv stem input, modeling_whisper.py:WhisperEncoder.forward). */
int32_t mm_transpose_pad(const void* x, int32_t B, int32_t C, int32_t T, int32_t pad, void* out, void* stream);
/* y[r,:] = x[r,:] + add[r % add_rows,:]  (bf16; CLIP class/position embeddings, video sinusoid PE modeling.py:1108-1118) */
int32_t mm_add_rows(const void* x, int64_t ldx, const void* add, int64_t lda, int32_t add_rows, void* y, int64_t ldy,
                    int32_t rows, int32_t cols, void* stream);
/* bf16 rows -> fp16 rows (modal features entering the fp16 alignment chain; exact within fp16's normal range) */
int32_t mm_cast_bf16_f16(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t rows, int32_t cols, void* stream);
/* generic strided 2-D copy of bf16 rows (concats, CLS drop) */
int32_t mm_copy_rows(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t rows, int32_t cols, void* stream);

/* ------------------------------------------------------------------------------------------------ fused alignment attention
 * The cross-modal alignment attention of reference modeling.py:986-987 / 1007-1008 / 1025-1026
 * (nn.MultiheadAttention with K = V = the whole embedding table, add_bias_kv, add_zero_attn; torch functional.py:6531-6672)
 * in ABSORBED form (SURVEY.md §7): for the R = H * Nq per-head query rows q~ = (q_h / sqrt(hd)) W_k[h] (fp16, width E)
 *     out[r, :]      = sum_{v < V} P[r, v] * table[v, :]                               (fp16, R x E; "ctx~")
 *     P[r, :]        = softmax over the S = V + 2 keys of { q~[r] . table[v] + row_bias[r] (v < V), extra[r], 0 }
 *     p_sum_real[r]  = sum_{v < V} P[r, v]        p_extra[r] = P of the appended bias_k key
 * ONE persistent kernel: phase 1 streams K-major table tiles through TMA into wgmma (S = q~ . table^T) and its
 * epilogue writes the un-normalised probabilities once, in fp16 (no fp32 score tensor, no softmax kernel); phase 2
 * streams the SAME table rows as an MN-major operand (O = P' . table) and normalises in its epilogue.  The caller
 * finishes with ctx_h = ctx~_h W_v[h]^T + p_sum_real * b_v[h] + p_extra * bias_v[h] (mm_gemm_fwd with row-scaled biases).
 * row_bias[r] = q_h . b_k[h] / sqrt(hd) and extra[r] = q_h . bias_k[h] / sqrt(hd) are read at index r * stat_stride.
 * P: scratch fp16 [R][ldp], ldp >= V rounded up to 8.  workspace: mm_align_workspace_bytes(R, V) bytes, 16-byte aligned
 * (zeroed by the call).  mode 0: one cooperative launch with grid-wide barriers between the phases; mode 1: the same
 * kernel launched three times in stream order (phase 1, conditional redo, phase 2). */
typedef struct mm_align_args {
  const void* table; /* fp16 [V][ldt] (exact fp16 copy of the bf16 embedding table) */
  int32_t V, E;
  int64_t ldt;
  const void* qt; /* fp16 [R][ldq] */
  int32_t R;
  int64_t ldq;
  const float* row_bias;
  const float* extra;
  int64_t stat_stride;
  void* out; /* fp16 [R][ldo] */
  int64_t ldo;
  float* p_sum_real;
  float* p_extra;
  void* P;
  int64_t ldp;
  void* workspace;
  int32_t mode;
  float* inv_l; /* optional fp32 [R]: 1 / softmax denominator, so that P = P' * inv_l (kept for the backward pass) */
} mm_align_args;
int32_t mm_align_fwd(const mm_align_args* args, void* stream);
int64_t mm_align_workspace_bytes(int32_t R, int32_t V);

/* ------------------------------------------------------------------------------------------------ decode (generate branch)
 * Greedy decoding behind inputs['inference'] = True (reference modeling.py:954-960 -> HF generate, vendored KV-cache
 * logic modeling.py:190-195).  mm_kv_append copies the K and V thirds of a fused [q|k|v] activation (rows (b, t),
 * row stride ld_qkv) into a per-layer cache (B, Tmax, 2, E) at time positions t0 .. t0 + T_new - 1.
 * mm_argmax_rows: out[r] = argmax_c logits[r, c] (lowest index on ties), bf16 logits, int64 out. */
int32_t mm_kv_append(const void* qkv, int64_t ld_qkv, int32_t B, int32_t T_new, int32_t E, void* cache, int32_t Tmax,
                     int32_t t0, const int32_t* t0_dev, void* stream); /* t0_dev != NULL overrides t0 with a device int */
int32_t mm_argmax_rows(const void* logits, int64_t ld, int32_t rows, int32_t V, int64_t* out, void* stream);
/* The int8 KV cache of the generate branch (same reference KV-cache logic, modeling.py:190-195, with K / V stored in int8).
 * Each cached key vector and each cached value vector of one token and one head (hd = 128 elements) is quantized on its
 * own.  v is the vector as the 16-bit cache would store it (keys after RoPE, rounded to the activation format):
 *   s = fp32(max_d |v_d|) / 127 (IEEE division),  q_d = clamp(rint(v_d / s), -127, 127) (IEEE division, ties to even),
 *   q = 0 where s = 0;  the dequantized value is the fp32 product q_d * s.
 * Layout per layer: cache int8 (B, Tmax, 2, E), indexed as the 16-bit cache; cache_scale fp32 (B, 2, H, Tmax), so one head's
 * scales run contiguously along the key axis.
 * mm_kv_append_i8: mm_kv_append's copy with that quantization (same arguments plus cache_scale; t0_dev overrides t0). */
int32_t mm_kv_append_i8(const void* qkv, int64_t ld_qkv, int32_t B, int32_t T_new, int32_t E, int8_t* cache,
                        float* cache_scale, int32_t Tmax, int32_t t0, const int32_t* t0_dev, void* stream);
/* mm_attn_decode_i8: one query row per (b, h) over the int8 cache (the decode step's attention, no mask):
 * out[b, h] = softmax_t(scale * s_k[t] * sum_d q_d kq[t, d]) . (s_v[t] vq[t]) over keys t < Tk, with Tk = min(*tk_dev, Tk)
 * when tk_dev is given (so a captured graph reads the count).  q 16-bit, element (b, h, d) at q[b * q_bs + h * 128 + d];
 * out likewise with o_bs.  Keys at or past the count are never read (neither values nor scales).  The keys are split over
 * CTAs by a layout that depends only on (B, H, Tmax, SM count); each split keeps its running max, sum and output in fp32 and
 * a second kernel merges the splits in a fixed order, so results are deterministic.  workspace: fp32, at least
 * mm_attn_decode_i8_workspace_bytes(B, H, Tmax) bytes.  No key: zeros. */
int32_t mm_attn_decode_i8(const void* q, int64_t q_bs, const int8_t* cache, const float* cache_scale, void* out,
                          int64_t o_bs, int32_t B, int32_t H, int32_t Tmax, int32_t Tk, const int32_t* tk_dev, float scale,
                          float* workspace, int64_t workspace_bytes, void* stream);
int64_t mm_attn_decode_i8_workspace_bytes(int32_t B, int32_t H, int32_t Tmax);
/* mm_sample_rows: the next token of HF generate's decoding step (reference modeling.py:959 -> llm.generate with
 * llm.generation_config): RepetitionPenaltyLogitsProcessor -> TemperatureLogitsWarper -> TopKLogitsWarper ->
 * TopPLogitsWarper -> softmax -> multinomial, in fp32 on the 16-bit logits (rows, V), row stride ld, V <= 49152.
 * seen: rows x ceil(V/32) uint32 bitmap of the tokens generated so far (the penalty's input_ids); the emitted token's bit
 * is set.  top_k 0 = off, top_p 1 = off.  Top-k keeps scores >= the k-th largest; top-p removes token i iff the kept
 * mass of all tokens with probability <= p_i is <= 1 - top_p (HF's ascending cumsum rule with tied probabilities
 * resolved together; the largest token always stays).  Draw: u = (w >> 8) * 2^-24, w = word 0 of
 * philox4x32_10(key = *seed_dev, counter = (*step_dev, row, 16, 0)); the token is the first kept one, in id order,
 * whose cumulative unnormalised mass exceeds u * Z.  do_sample = 0: greedy search on the penalised scores (argmax,
 * lowest index on ties; temperature / top-k / top-p unused, seed_dev / step_dev may be NULL).  The result is a pure
 * function of the inputs (no order-dependent arithmetic). */
int32_t mm_sample_rows(const void* logits, int64_t ld, int32_t rows, int32_t V, uint32_t* seen, float repetition_penalty,
                       float temperature, int32_t top_k, float top_p, int32_t do_sample, const uint64_t* seed_dev,
                       const int32_t* step_dev, int64_t* out, void* stream);
/* Fused tail of a split-K thin (decode) GEMM: part fp32 [splits][N][ldp] holds W_s x_s^T per K slice (mm_gemm_fwd with
 * the operands swapped, batch = splits, fp32 out).  Splitting K lets the 32-tile o_proj / down_proj grids of a decode step
 * cover all 132 SMs (weight streaming); one launch per GEMM finishes the sum and the ops around it (a decode step is
 * launch-bound):
 *   MM_THIN_RES     out = rs * sum_s part + residual; sumsq_out (optional, [M][N/32]) = per-(row, 32-column) sums of squares
 *                   of the stored values, the next RMSNorm's statistic (LlamaRMSNorm modeling.py:311-319)
 *   MM_THIN_SWIGLU  out[m][32q+i] = silu(gate) * up from the [32 gate | 32 up]-interleaved product (modeling.py:139-140)
 *   MM_THIN_QKV     N = 3E: rotate-half RoPE (modeling.py:83-91) on q and k in fp32, q -> out[m][0..E), k / v -> the
 *                   layer's KV cache (B, Tmax, 2, E) at slot t0 (*t0_dev if given), row m = sample m (modeling.py:190-195)
 * rs = row_scale[m] | rsqrt(sum_j rs_sumsq[m][j] / rs_K + rs_eps) | 1. */
enum { MM_THIN_RES = 0, MM_THIN_SWIGLU = 1, MM_THIN_QKV = 2 };
typedef struct mm_thin_args {
  const float* part;       /* [splits][N][ldp] fp32 */
  int32_t splits, N, M, ldp, mode;
  const float* row_scale;  /* [M] or null */
  const float* rs_sumsq;   /* [M][rs_parts] or null */
  int32_t rs_parts, rs_K;
  float rs_eps;
  const void* residual;    /* [M][ldr] 16-bit or null (MM_THIN_RES) */
  int64_t ldr;
  void* out;
  int64_t ldo;
  float* sumsq_out;
  const float* rope_cos;   /* MM_THIN_QKV: (T, 64) fp32 tables; row = *pos_dev (0 if null) */
  const float* rope_sin;
  const int32_t* pos_dev;
  int32_t E;
  void* cache;
  int32_t Tmax, t0;
  const int32_t* t0_dev;
} mm_thin_args;
int32_t mm_thin_fused(const mm_thin_args* args, void* stream);
/* mm_thin_fused_kv_i8: the MM_THIN_QKV tail with an int8 cache (see mm_kv_append_i8).  k / v are rounded to 16 bits as
 * MM_THIN_QKV stores them, then each head vector is quantized into args->cache (int8 (B, Tmax, 2, E)) and cache_scale
 * (fp32 (B, 2, H, Tmax)) at slot t0 (*t0_dev if given); q rows -> out in 16 bits as in MM_THIN_QKV.  args->mode must be
 * MM_THIN_QKV. */
int32_t mm_thin_fused_kv_i8(const mm_thin_args* args, float* cache_scale, void* stream);
/* In-place rotate-half RoPE (head_dim 128, apply_rotary_pos_emb modeling.py:83-91) on the first rot_cols columns of each
 * row; position of row r = (*pos_dev if given) + r % rope_T.  The training step's RoPE backward calls it with the sin
 * table negated (the rotation is orthogonal: its transpose is the rotation by -theta). */
int32_t mm_rope_rows(void* x, int64_t ld, int32_t rows, int32_t rot_cols, const float* cos_t, const float* sin_t,
                     int32_t rope_T, const int32_t* pos_dev, void* stream);

/* ------------------------------------------------------------------------------------------------ loss
 * Shifted cross entropy of LlamaForCausalLM.forward modeling.py:600-610: logits bf16 (B, T, V), labels int64 (B, T);
 * position t predicts labels[t+1]; ignore_index -100; writes loss_sum[0] (fp32) and n_valid[0] (int32);
 * both must be zeroed by the caller. */
int32_t mm_ce_loss(const void* logits, const int64_t* labels, int32_t B, int32_t T, int32_t V, float* loss_sum,
                   int32_t* n_valid, void* stream);

/* ------------------------------------------------------------------------------------------------ training step
 * Backward halves of the HBM-bound ops + the optimizer (SURVEY.md §8f rank 1).  The reference trains through autograd of
 * modeling.py driven by llm_trainer.py:184-188 (compute_loss -> backward) with AdamW (train.sh, fp32 master weights in
 * DeepSpeed).  All contractions of the backward pass are mm_gemm_fwd calls (dX: MN-major B; dW: MN-major A and B).
 *
 * mm_rmsnorm_bwd: y = x * rstd * g (LlamaRMSNorm modeling.py:311-319).  dx = rstd*(g*dy) - rstd^3/cols * x * sum(g*dy*x)
 *   (+ dres when given: the residual branch's gradient), dg[c] += sum_r dy*x*rstd in fp32: through dg_partials
 *   ([mm_rmsnorm_bwd_parts(rows)][cols] fp32 workspace: per-CTA column sums reduced in a fixed order — deterministic, and
 *   no grid-size-way atomic contention on `cols` addresses) or, when dg_partials is null, with atomics. */
int32_t mm_rmsnorm_bwd_parts(int32_t rows);
int32_t mm_rmsnorm_bwd(const void* dy, const void* x, const float* rstd, const void* g, const void* dres, void* dx,
                       float* dg, float* dg_partials, int32_t rows, int32_t cols, void* stream);
/* LlamaMLP modeling.py:139-140 on separate gate / up activations: h = silu(gate) * up over n contiguous elements. */
int32_t mm_swiglu_fwd(const void* gate, const void* up, void* h, int64_t n, void* stream);
int32_t mm_swiglu_bwd(const void* dh, const void* gate, const void* up, void* dgate, void* dup, int64_t n, void* stream);
/* Attention backward through the softmax (LlamaAttention modeling.py:197-215; nn.MultiheadAttention): S = q.k^T (pre-scale)
 * and dP = dO.v^T, fp32 [B][H][Tq][ld]; writes P = softmax(scale*S + mask) and dS = scale * P * (dP - sum_j P_j dP_j) as
 * bf16 with the same layout.  Masks as in mm_attn_fwd. */
int32_t mm_attn_softmax_bwd(const float* S, const float* dP, void* P, void* dS, int32_t B, int32_t H, int32_t Tq,
                            int32_t Tk, int64_t ld, float scale, int32_t causal, const int32_t* key_mask, float p_drop,
                            const uint64_t* seed_dev, uint32_t sid, void* stream);
/* Training-mode attention dropout (reference: nn.MultiheadAttention(dropout=0.1), modeling.py:879-909; torch drops the
 * softmax probabilities, functional.py:6640-6645).  The mask is a pure function of (*seed_dev, sid, row, column) through
 * Philox4x32-10 (csrc/philox.cuh): forward and backward kernels regenerate it, nothing is stored; `seed_dev` is a DEVICE
 * 64-bit seed so a captured CUDA graph draws a fresh mask per replay, `sid` separates the dropout sites.  p_drop == 0
 * switches dropout off (seed_dev may be null).  With p_drop > 0, mm_attn_softmax_bwd uses dP <- m . dP and writes Pd = m . P.
 * mm_attn_softmax_fwd: S fp32 [B][H][Tq][ld] -> Pd = dropout(softmax(scale * S + mask)) bf16, same layout. */
int32_t mm_attn_softmax_fwd(const float* S, void* P, int32_t B, int32_t H, int32_t Tq, int32_t Tk, int64_t ld, float scale,
                            int32_t causal, const int32_t* key_mask, float p_drop, const uint64_t* seed_dev, uint32_t sid,
                            void* stream);
/* Dropout of the alignment attention's probabilities (forward): P' (un-normalised fp16, R x ldp) -> Pm (kept entries,
 * unscaled), rs = (1/l)/(1-p), p_sum_real_d = rs * sum_v Pm_v, p_extra_d = m_V * p_extra (column V = the bias_k key). */
int32_t mm_align_dropout_fwd(const void* P_unnorm_f16, void* Pm_f16, int64_t ldp, const float* inv_l, const float* p_extra,
                             float* rs, float* p_sum_real_d, float* p_extra_d, int32_t R, int32_t V, float p_drop,
                             const uint64_t* seed_dev, uint32_t sid, void* stream);
/* The multipliers themselves (fp32: 0 or 1/(1-p)) of a rows x cols block of stream `sid` — for tests / debugging. */
int32_t mm_dropout_mask(float* out, int64_t ld, int32_t rows, int32_t cols, float p_drop, const uint64_t* seed_dev,
                        uint32_t sid, void* stream);
/* Gradient of mm_ce_loss w.r.t. the logits (modeling.py:600-610), times grad_scale (* *grad_scale_dev when given: the
 * upstream gradient of the loss as a device scalar, so the launch is CUDA-graph capturable) / n_valid; may run in place. */
int32_t mm_ce_bwd(const void* logits, const int64_t* labels, void* dlogits, int32_t B, int32_t T, int32_t V,
                  const int32_t* n_valid, float grad_scale, const float* grad_scale_dev, void* stream);
/* Gradient of mm_embed_gather: dtable[ids[i], :] += dx[i, :] (bf16x2 atomics; half2 atomics in fp16). */
int32_t mm_embed_scatter_add(const void* dx, int64_t ldx, const int64_t* ids, int64_t n, int32_t dim, int32_t vocab,
                             void* dtable, void* stream);
/* out[c] += sum_r x[r, c]  (bias gradients; fp32 atomics) */
int32_t mm_colsum(const void* x, int64_t ldx, int32_t rows, int32_t cols, float* out, void* stream);
/* Fused AdamW step on one parameter tensor: 16-bit working copy p and gradient g in the activation format (g times
 * grad_scale), fp32 master / m / v.  The bias corrections use `step`, or the device int *step_dev when given
 * (graph-replayed training steps).  grad_mult_dev (nullable): a device fp32 multiplier that replaces grad_scale — the
 * unscale-and-clip factor of mm_loss_scale_update (DeepSpeed FP16_Optimizer.unscale_and_clip_grads).  skip_dev
 * (nullable): a device int; when non-zero the launch writes nothing (p, master, m, v unchanged: the overflow-skipped
 * step of DeepSpeed's fp16 optimizer).  With both null the behaviour is that of ABI 3.  lr_dev (nullable, ABI 6): a device
 * fp32 lr that replaces `lr` — the output of mm_lr_schedule; every AdamW kernel (8-wide, scalar, host-state) reads it
 * alike.  With lr_dev null the results are those of ABI 5, bit for bit. */
int32_t mm_adamw(void* p, const void* g, float* master, float* m, float* v, int64_t n, float lr, float beta1, float beta2,
                 float eps, float weight_decay, int32_t step, const int32_t* step_dev, float grad_scale,
                 const float* grad_mult_dev, const int32_t* skip_dev, const float* lr_dev, void* stream);
/* AdamW state in page-locked host memory (DeepSpeed's offload_optimizer {device: cpu, pin_memory: true}, but updated by
 * the GPU: no CPU execution path).  mm_host_alloc allocates exactly `bytes` with cudaHostAllocMapped |
 * cudaHostAllocPortable and returns the host pointer and its device alias (cudaHostGetDevicePointer); it fails when the
 * current device cannot map host memory.  mm_host_free releases a block by its host pointer.
 * mm_adamw_host: mm_adamw's arguments and arithmetic (bit-identical results: one shared per-element update), with
 * master / m / v device aliases of mm_host_alloc memory (16-byte aligned) and p / g in device memory (8-byte aligned).
 * The launch is bound by the PCIe link: lane-contiguous 16-byte accesses, 24 B of host traffic per element. */
int32_t mm_adamw_host(void* p, const void* g, float* master, float* m, float* v, int64_t n, float lr, float beta1,
                      float beta2, float eps, float weight_decay, int32_t step, const int32_t* step_dev, float grad_scale,
                      const float* grad_mult_dev, const int32_t* skip_dev, const float* lr_dev, void* stream);
int32_t mm_host_alloc(int64_t bytes, void** host_ptr, void** dev_ptr);
int32_t mm_host_free(void* host_ptr);

/* ------------------------------------------------------------------------------------------------ loss scaling / clipping
 * fp16 training with dynamic loss scaling and global gradient-norm clipping, on the device and free of host syncs (the
 * whole optimizer step stays CUDA-graph capturable).  Reference: train.sh `--fp16 True` with DeepSpeed's fp16 optimizer,
 * configs/deepspeed_config.json "fp16" block (loss_scale 0 = dynamic, initial_scale_power 16, loss_scale_window 1000,
 * hysteresis 2, min_loss_scale 1) and "gradient_clipping": "auto" = HF TrainingArguments.max_grad_norm (1.0).
 *
 * mm_grad_sumsq: *out += sum_i g[i]^2 (fp32) over a flat 16-bit gradient buffer (fp16 != 0: IEEE half, else bf16; g
 *   16-byte aligned, 64-bit n).  Deterministic: the grid is fixed by (n, device), `partials` (mm_grad_sumsq_parts(n) fp32)
 *   holds one partial per CTA, summed in a fixed order.  A NaN / Inf element makes the result non-finite (overflow test).
 *   Several ranges can be summed into one scalar by successive calls (fixed order = deterministic total). */
int32_t mm_grad_sumsq_parts(int64_t n);
int32_t mm_grad_sumsq(const void* g, int64_t n, int32_t fp16, float* out, float* partials, void* stream);
/* Device-side state of the loss scaler (DeepSpeed DynamicLossScaler) and of the optimizer step it gates. */
typedef struct mm_loss_scale_state {
  float scale;                /* S: the loss is multiplied by S before backward */
  float inv_scale;            /* 1 / S */
  int32_t cur_iter;           /* optimizer steps seen (skipped ones included) */
  int32_t last_overflow_iter; /* -1 initially */
  int32_t cur_hysteresis;     /* overflows still tolerated before the scale is halved */
  int32_t skip;               /* 1: the latest step's gradients were non-finite; mm_adamw(skip_dev) writes nothing */
  float grad_mult;            /* per-element gradient multiplier of the latest step: 1 / (S * max(clip, 1)) */
  int32_t skipped;            /* skipped steps so far */
  int32_t step;               /* AdamW step counter (bias corrections), advanced on steps that are not skipped */
  float grad_norm;            /* unscaled global gradient norm of the latest step (non-finite on overflow) */
  int32_t reserved[2];
} mm_loss_scale_state;
/* mm_loss_scale_update: one single-thread launch after the gradient sum of squares, before the AdamW launches.
 *   overflow = !isfinite(*sumsq);  norm = sqrt(*sumsq) / S;
 *   grad_mult = 1 / (S * max((norm + 1e-6) / max_norm, 1))  (max_norm > 0: clipping on), else 1 / S;
 *   skip = overflow (counted in `skipped`), else step += 1;
 *   dynamic != 0: DynamicLossScaler.update_scale — on overflow, S = max(S / 2, min_scale) if hysteresis == 1 or
 *   cur_hysteresis == 1, else cur_hysteresis -= 1, and last_overflow_iter = cur_iter; without overflow, when
 *   (cur_iter - last_overflow_iter) % window == 0: cur_hysteresis = hysteresis, S *= 2.  At S == min_scale an overflow
 *   keeps S (a kernel cannot raise) and the step is skipped.  Then cur_iter += 1.  *sumsq is reset to 0. */
int32_t mm_loss_scale_update(mm_loss_scale_state* state, float* sumsq, float max_norm, int32_t dynamic, int32_t window,
                             int32_t hysteresis, float min_scale, void* stream);

/* ------------------------------------------------------------------------------------------------ learning-rate schedule
 * The lr of every AdamW step computed on the device from the AdamW step counter, so the whole step stays one CUDA graph
 * with no host sync.  Reference: train.sh `--learning_rate 3e-5 --warmup_ratio 0.03 --lr_scheduler_type cosine`; HF
 * Trainer builds the schedule (transformers.optimization get_*_schedule_with_warmup, a LambdaLR) and DeepSpeed steps it
 * only on steps it does not skip for overflow.
 *
 * mm_lr_schedule: one single-thread launch per optimizer step, AFTER mm_loss_scale_update (or the increment of the
 * caller's step counter when there is neither scaler nor clipping) and BEFORE the AdamW launches, which get lr_out as
 * their lr_dev.  With t = *step_dev (mm_loss_scale_state.step, the counter the bias corrections use: t-th applied update)
 * and n = max(t - 1, 0), in double:
 *   *lr_out = fp32(base_lr * lambda(n)),  W = warmup_steps, N = training_steps,
 *   kind 0 linear:                lambda = n / max(1, W) for n < W, else max(0, (N - n) / max(1, N - W))
 *   kind 1 cosine:                lambda = n / max(1, W) for n < W, else max(0, 0.5 (1 + cos(pi (n - W) / max(1, N - W))))
 *                                 (not clamped past N: it rises again, as HF's)
 *   kind 2 constant_with_warmup:  lambda = n / max(1, W) for n < W, else 1
 * The first applied update therefore runs at lr 0 when W > 0 (HF's LambdaLR): m and v move, master and p do not.  Skip
 * rule: an overflow-skipped step does not advance t, so it does not advance the schedule (the launch rewrites the lr of the
 * latest applied update, which the skipped AdamW launches do not use); after k skips the schedule runs k steps behind the
 * iteration count.  Gradient-accumulation micro-batches do not advance it either.  Arguments are checked before any CUDA
 * call: non-null pointers, kind in 0..2, 0 <= W <= N, N >= 1. */
int32_t mm_lr_schedule(const int32_t* step_dev, double base_lr, int32_t kind, int32_t warmup_steps, int32_t training_steps,
                       float* lr_out, void* stream);

/* Backward of the absorbed alignment attention through its (V + 2)-key softmax (reference: autograd of
 * nn.MultiheadAttention, modeling.py:986-987 / 1007-1008 / 1025-1026).  See train_kernels.cu for the formulas. */
int32_t mm_align_softmax_bwd(const float* G, int64_t ldg, const void* P_unnorm_f16, int64_t ldp, const float* inv_l,
                             const float* d_p_sum_real, const float* p_extra, const float* d_p_extra, float gscale,
                             void* P_bf16, void* dS_bf16, int64_t ldo, float* dstats, int32_t R, int32_t V, float p_drop,
                             const uint64_t* seed_dev, uint32_t sid, void* stream);
/* out[h*hd + d] += sum_n w[(h*Nq + n) * w_stride] * x[n, h*hd + d]; x bf16 (x_fp16 == 0) or fp16. */
int32_t mm_head_weighted_colsum(const void* x, int64_t ldx, int32_t x_fp16, const float* w, int64_t w_stride, int32_t Nq,
                                int32_t E, int32_t head_dim, float* out, void* stream);
/* Data gradient of the Conv1d down-sampler (col2im over overlapping token windows): dfeats[b,t,c] = sum over windows l
 * containing t of dwin[b*Lq + l][(t - l*ss)*C + c]; bf16 in / out. */
int32_t mm_window_gather_add(const void* dwin, int32_t B, int32_t N, int32_t C, int32_t Lq, int32_t kk, int32_t ss,
                             void* dfeats, void* stream);
int32_t mm_cast_f16_bf16(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t rows, int32_t cols, void* stream);

/* ------------------------------------------------------------------------------------------------ LoRA adapters
 * Low-rank adapters on a frozen nn.Linear (PEFT's LoraLayer.forward): y = x W^T + s * drop(x) A^T B^T, s = lora_alpha / r,
 * A (r, K), B (N, r), drop = inverted dropout with the Philox mask of csrc/philox.cuh (stream sid[j], the training step's
 * device seed; p = 0 or seed null: off).  The mask of input element (m, k) is that of mm_dropout_mask(row m, col k): the
 * backward pass regenerates it.  One launch serves n (1..MM_LORA_MAX) adapters of the same shapes; in the down and
 * dx-backward entries they share the input x (q / k / v, gate / up read it once).  Tensors are 16-bit in the activation
 * format unless marked fp32; rows are contiguous unless a leading dimension is given; 8 <= r <= 64, r % 8 == 0,
 * K % 8 == 0.  Every reduction is a fixed-order sum (per-CTA partials in `workspace`): results are deterministic.
 *   mm_lora_down    u[j] (M, r) fp32 = drop_j(x) A_j^T
 *   mm_lora_up      y[j] (M, N, ld ldy) <- round(rope(y[j] + s u[j] B_j^T)), in place.  With rope_cos / rope_sin (fp32
 *                   (T, 64) tables, position = row % rope_T) the rotate-half RoPE over 128-wide heads (pairs c, c + 64)
 *                   is applied in fp32 before the one rounding (N % 128 == 0): the adapted q / k projection.
 *   mm_lora_bwd_dy  with dy = y[j] (M, N, ld ldy): g[j] (M, r) fp32 = s dy B_j;  dB[j] (N, r) (+)= s dy^T u[j]
 *   mm_lora_bwd_x   dA[j] (r, K) (+)= g[j]^T drop_j(x);  dx (M, K, ld lddx) <- round(dx + sum_j drop_j(g[j] A_j)), in place
 * accumulate[j] != 0 adds the gradient of adapter j to dA[j] / dB[j] (fp32 sum, one rounding), else overwrites them.
 * mm_lora_workspace_bytes: the fp32 workspace `entry` (2 = bwd_dy, 3 = bwd_x; 0 otherwise) needs for these shapes. */
#define MM_LORA_MAX 3
typedef struct mm_lora_args {
  int32_t n, M, K, N, r;
  float scaling, p_drop;
  const uint64_t* seed_dev;
  uint32_t sid[MM_LORA_MAX];
  const void* x;
  int64_t ldx;
  const void* A[MM_LORA_MAX];
  const void* B[MM_LORA_MAX];
  float* u[MM_LORA_MAX];
  void* y[MM_LORA_MAX];
  int64_t ldy;
  const float* rope_cos;
  const float* rope_sin;
  int32_t rope_T;
  float* g[MM_LORA_MAX];
  void* dA[MM_LORA_MAX];
  void* dB[MM_LORA_MAX];
  int32_t accumulate[MM_LORA_MAX];
  void* dx;
  int64_t lddx;
  float* workspace;
  int64_t workspace_bytes;
} mm_lora_args;
int32_t mm_lora_down(const mm_lora_args* args, void* stream);
int32_t mm_lora_up(const mm_lora_args* args, void* stream);
int32_t mm_lora_bwd_dy(const mm_lora_args* args, void* stream);
int32_t mm_lora_bwd_x(const mm_lora_args* args, void* stream);
int64_t mm_lora_workspace_bytes(const mm_lora_args* args, int32_t entry);

/* ------------------------------------------------------------------------------------------------ int8 decoder weights
 * Weight-only int8 with one fp32 scale per output row (csrc/quant.cu).
 *
 * mm_quantize_rows_int8: w (rows, K) with row stride ldw, format w_format (0 bf16, 1 fp16, 2 fp32) ->
 *   s[n] = fp32(max_k |w[n][k]|) / 127 (IEEE division), q[n][k] = clamp(rint(fp32(w[n][k]) / s[n]), -127, 127) (round half
 *   to even), q = 0 where s = 0.  q is (rows, K) contiguous, s is [rows].
 *
 * An mm_w8_matrix describes a FUSED weight matrix (N, K) whose rows live in up to MM_W8_MAX_SRC separate int8 matrices: the
 * device table `chunks` [N / 32][2] names, for fused rows 32c .. 32c + 31, the source j and its first row (the decoder's
 * [q; k; v] concatenation and [32 gate | 32 up] interleave need no copy of the weights).  Source j is q[j] (rows[j], K)
 * contiguous with scales scale[j] [rows[j]] (rows[j] % 32 == 0).  gain: [K] 16-bit (activation format) RMSNorm gain, or null.  N % 64 == 0,
 * K % 16 == 0.
 *
 * mm_dequant_rows: out (N, K, row stride ldo, activation format) = round16(fp32(fp32(q s) g)) (without gain:
 *   round16(fp32(q s))) — the fused 16-bit weight the prefill GEMMs read.
 * mm_gemm_w8_thin: the split-K partial sums of a decode GEMM for the mm_thin_fused tail,
 *   part[s][n][m] (row stride ldp >= M) = s_n * sum_{k in slice s} q[n][k] x~[m][k],   x~ = round16(x[m][k] g[k]),
 *   x (M <= 64, K) 16-bit with row stride ldx (ldx % 8 == 0).  Slice s covers the 128-column stages
 *   [s ns / splits, (s + 1) ns / splits), ns = ceil(K / 128); 1 <= splits <= ns.  xs_work: 16-bit scratch of
 *   M * 128 * ns elements.  When the x~ rows of the longest slice (M rounded up to 8 / 16 / 32 / 64, 256 bytes per row per
 *   stage) fit MM_W8_XS_BYTES they are staged in shared memory once per CTA; otherwise x~ is first written to xs_work and
 *   streamed through the pipeline with the weights (one more launch).
 * A chunk-table entry that does not name 32 rows of a present source contributes zero rows. */
#define MM_W8_MAX_SRC 3
#define MM_W8_XS_BYTES 49152
typedef struct mm_w8_matrix {
  const int8_t* q[MM_W8_MAX_SRC];
  const float* scale[MM_W8_MAX_SRC];
  int32_t rows[MM_W8_MAX_SRC];
  const int32_t* chunks;
  int32_t N, K;
  const void* gain;
} mm_w8_matrix;
int32_t mm_quantize_rows_int8(const void* w, int64_t ldw, int32_t w_format, int32_t rows, int32_t K, int8_t* q, float* scale,
                              void* stream);
int32_t mm_dequant_rows(const mm_w8_matrix* w, void* out, int64_t ldo, void* stream);
int32_t mm_gemm_w8_thin(const mm_w8_matrix* w, const void* x, int64_t ldx, int32_t M, float* part, int32_t splits,
                        int32_t ldp, void* xs_work, void* stream);

/* ------------------------------------------------------------------------------------------------ FP8 (e4m3) decoder
 * Per-row e4m3 weights AND activations for the decoder's prefill GEMMs (csrc/quant.cu, csrc/gemm_wgmma.cu).
 *
 * mm_quantize_rows_e4m3: x (rows, K) with row stride ldx, format x_format (0 bf16, 1 fp16, 2 fp32), optional gain [K] in
 *   the activation format -> v = fp32(x) * fp32(g) (v = fp32(x) without gain),
 *   s[r] = fp32(max_k |v[r][k]|) / 448 (IEEE division),  q[r][k] = e4m3(v[r][k] / s[r]) (IEEE division, round to nearest
 *   even, saturated to +-448: cvt.rn.satfinite), q = 0 where s = 0.  q (rows, K) bytes with row stride ldq; K % 16 == 0,
 *   x, gain and q 16-byte aligned, ldx a whole number of 16-byte units, ldq % 16 == 0.  Deterministic, no host
 *   synchronisation.
 *
 * mm_gemm_e4m3_fwd: mm_gemm_fwd's epilogues on an e4m3 product,
 *   C = epilogue((acc[m][n] * a_scale[m]) * s_w[n]),  acc = sum_k qa[m][k] qw[n][k] (fp32),
 *   with A = args->A the e4m3 activation rows (M, K) (row stride args->lda bytes, lda % 16 == 0) and the weight the e4m3
 *   mm_w8_matrix `w` (its q[] hold e4m3 bytes; gathered through w.chunks, no fused copy; w.gain must be null; w.N ==
 *   args->N, w.K == args->K).  Every other field of args means what it means for mm_gemm_fwd, except: args->B / ldb /
 *   a_fp16 / b_fp16 and the stream-K workspace are ignored; no batching, no c_trans, no MN-major operands; K % 128 == 0,
 *   N % 128 == 0.  The main loop accumulates each 128-deep k-block in a fresh register tile and adds it to fp32 master
 *   accumulators (promotion every four k32 MMAs); `unpromoted` = 1 lets the MMAs accumulate all of K in place instead
 *   (a comparison instance for tests).  The variant is always MM_GEMM_KERNEL_CONSUMER_EPILOGUE with block_n = 128.
 * mm_gemm_e4m3_plan: the launch mm_gemm_e4m3_fwd would make for these arguments (no memory is touched, no GPU needed).
 * mm_gemm_e4m3_thin: mm_gemm_w8_thin with e4m3 weight bytes (converted exactly to the activation format in registers):
 *   part[s][n][m] = s_n * sum_{k in slice s} e4m3(q[n][k]) x~[m][k], x~ = round16(x[m][k] g[k]); same arguments. */
typedef struct mm_gemm_e4m3_args {
  const float* a_scale;   /* [M] fp32 per-row scales of A */
  mm_w8_matrix w;         /* the weight: e4m3 sources, per-row fp32 scales, chunk table */
  int32_t unpromoted;
} mm_gemm_e4m3_args;
int32_t mm_quantize_rows_e4m3(const void* x, int64_t ldx, int32_t x_format, int32_t rows, int32_t K, const void* gain,
                              uint8_t* q, int64_t ldq, float* scale, void* stream);
int32_t mm_gemm_e4m3_fwd(const mm_gemm_args* args, const mm_gemm_e4m3_args* e, void* stream);
int32_t mm_gemm_e4m3_plan(const mm_gemm_args* args, const mm_gemm_e4m3_args* e, mm_gemm_schedule* plan);
int32_t mm_gemm_e4m3_thin(const mm_w8_matrix* w, const void* x, int64_t ldx, int32_t M, float* part, int32_t splits,
                          int32_t ldp, void* xs_work, void* stream);

/* ------------------------------------------------------------------------------------------------ gradient all-reduce
 * The one collective of the path: the data-parallel gradient all-reduce of the training step (reference: DeepSpeed ZeRO-3
 * reduce-scatter / all-gather, configs/deepspeed_config.json:22-41; north_star: "a single NCCL all-reduce on gradients").
 * NCCL is bound at run time (dlopen); one communicator per process (one process per GPU).  Bootstrap: rank 0 calls
 * mm_nccl_unique_id, ships the 128 bytes to the other ranks (any channel: torch.distributed store, MPI, a file), every
 * rank calls mm_nccl_init.  mm_nccl_allreduce is in place, asynchronous on `stream`; dtype 0 = bf16, 1 = fp32, 2 = fp16
 * (the gradients of an fp16 model: the loss-scale overflow test runs after the all-reduce, so every rank skips alike);
 * average != 0 divides by the group size (ncclAvg). */
int32_t mm_nccl_unique_id(void* out128);
int32_t mm_nccl_init(const void* id128, int32_t world, int32_t rank);
int32_t mm_nccl_allreduce(void* buf, int64_t count, int32_t dtype, int32_t average, void* stream);
int32_t mm_nccl_destroy(void);

/* ------------------------------------------------------------------------------------------------ input pipeline
 * Device-side replacement of the per-sample host work in LLMTrainer.get_self_inputs (llm_trainer.py:306-381).
 *
 * mm_image_preprocess: `_transform(224)` of llm_trainer.py:151-158 on ONE decoded 8-bit RGB image (HWC, row stride ld bytes):
 * Pillow's two-pass antialiased bicubic resize with its 22-bit fixed-point coefficients (tables built by the host with
 * Pillow's arithmetic, restricted to the centre-crop window), then ToTensor + Normalize.  row0 / n_rows: source rows the
 * vertical taps of the cropped output need (tmp holds n_rows x out_w x 3 bytes).  out: (3, out_h, out_w) bf16 or fp32;
 * out_u8 (optional, HWC) receives the 8-bit resized + cropped image (bit-exact with PIL). */
typedef struct mm_image_args {
  const void* src;
  int64_t ld;
  int32_t row0, n_rows;
  int32_t out_h, out_w;
  const int32_t* bounds_h; /* [out_w][2] = (xmin, count) */
  const int32_t* kk_h;     /* [out_w][ksize_h] */
  int32_t ksize_h;
  const int32_t* bounds_v; /* [out_h][2] */
  const int32_t* kk_v;     /* [out_h][ksize_v] */
  int32_t ksize_v;
  float mean[3], std[3];
  void* tmp;
  void* out;
  int32_t out_fp32;
  void* out_u8;
} mm_image_args;
int32_t mm_image_preprocess(const mm_image_args* args, void* stream);
/* whisper.pad_or_trim + whisper.log_mel_spectrogram (llm_trainer.py:338-345) of ONE clip: pcm fp32 [n_samples] at 16 kHz ->
 * (80, 3000) bf16 / fp32.  basisT: fp32 [400][2][208] windowed DFT basis (Hann folded in; cos, -sin; bin index
 * contiguous); mel: fp32 [80][201] filter bank; logspec: scratch fp32 [80][3000]; max_scratch: 4 bytes. */
int32_t mm_log_mel(const float* pcm, int32_t n_samples, const float* basisT, const float* mel, float* logspec,
                   void* max_scratch, void* out, int32_t out_fp32, void* stream);

/* mm_jpeg_decode: a batch of sequential Huffman JPEG files (8-bit, grayscale or YCbCr with luma sampling 1x1 / 2x1 / 2x2
 * and chroma 1x1, one scan) decoded bit-exactly as libjpeg-turbo does with its defaults (ISLOW IDCT, fancy upsampling,
 * fixed-point YCbCr -> RGB), in three kernels:
 *   1. entropy decode, one thread per entropy-coded segment (a restart interval, or the whole scan): int16 coefficients,
 *      natural order, per component in block order (coef + coef_off[c], block (by, bx) at (by * bw[c] + bx) * 64);
 *   2. dequantise + ISLOW IDCT: uint8 component planes padded to whole blocks (planes + plane_off[c], row stride bw[c] * 8);
 *   3. fancy upsampling + YCbCr -> RGB: HWC uint8 at out + out_off, row stride out_ld bytes.
 * The host parses the markers and packs every file's scan bytes into `data` and the descriptors below into device memory.
 * Whatever the bytes, the kernels read inside their segment and write inside their image's buffers; an inconsistency sets
 * bits of status[image] (zeroed by the call): 1 invalid Huffman code, 2 coefficient run past 63, 4 segment ends early,
 * 8 bytes left over after a segment's last MCU, 16 bad byte stuffing, 32 descriptor out of range.  max_blocks / max_pixels:
 * the batch's largest component block count and largest width * height (launch geometry). */
typedef struct mm_jpeg_image {
  int32_t width, height;
  int32_t n_comp;             /* 1 or 3 */
  int32_t hmax, vmax;         /* luma sampling factors; chroma is 1 x 1 (1 x 1 for grayscale) */
  int32_t mcus_x, mcus_y;
  int32_t seg0, n_seg;        /* segments[seg0 .. seg0 + n_seg) */
  int32_t bw[3], bh[3];       /* blocks per row / column of each component (whole MCUs) */
  int32_t huff_dc[3], huff_ac[3]; /* indices into huff[] */
  int32_t quant[3];           /* indices into quant[] */
  int64_t coef_off[3];        /* int16 elements */
  int64_t plane_off[3];       /* bytes */
  int64_t out_off, out_ld;    /* bytes */
} mm_jpeg_image;
typedef struct mm_jpeg_segment {
  int64_t offset;             /* bytes into data, markers excluded */
  int32_t n_bytes;
  int32_t image;
  int32_t mcu0, n_mcu;
} mm_jpeg_segment;
typedef struct mm_jpeg_huff {   /* libjpeg's derived table (jdhuff.c jpeg_make_d_derived_tbl) */
  int32_t maxcode[18];          /* largest code of each length, -1 if none; [17] = 0xFFFFF */
  int32_t valoffset[18];        /* huffval index = code + valoffset[length] */
  uint16_t look[256];           /* 8-bit lookahead: (length << 8) | symbol, 0 = code longer than 8 bits */
  uint8_t huffval[256];
} mm_jpeg_huff;
typedef struct mm_jpeg_args {
  int32_t n_images, n_segments, n_huff, n_quant;
  const uint8_t* data;
  int64_t data_bytes;
  const mm_jpeg_image* images;
  const mm_jpeg_segment* segments;
  const mm_jpeg_huff* huff;
  const uint16_t* quant;      /* [n_quant][64], natural order */
  int16_t* coef;
  int64_t coef_elems;
  uint8_t* planes;
  int64_t plane_bytes;
  uint8_t* out;
  int64_t out_bytes;
  int32_t* status;            /* [n_images] */
  int32_t max_blocks, max_pixels;
} mm_jpeg_args;
int32_t mm_jpeg_decode(const mm_jpeg_args* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MACAW_B200_H_ */
