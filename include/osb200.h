/*
 * osb200 — C ABI of the H100-native (sm_90a) hot path for Open-Sora's denoiser blocks and
 * causal 3D VAE.  This header is the drop-in boundary: plain pointers and sizes, no torch
 * types, no exceptions.  Each entry point cites the reference call site (path:line under the
 * reference checkout hpcaitech/Open-Sora @ 7ad6a96) whose arithmetic it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch); the library never
 *     allocates or frees device memory and keeps no pointer past the call;
 *   - all work is enqueued on `stream` (a cudaStream_t / CUstream passed as void*); there are
 *     no hidden synchronisations, so every call is CUDA-graph capturable;
 *   - return value: 0 on success, negative osb_status on failure; osb_last_error() returns a
 *     thread-local, human readable description of the last failure;
 *   - bf16 tensors are row-major with an explicit leading dimension in ELEMENTS; all leading
 *     dimensions and base pointers of GEMM operands must be 16-byte aligned.
 */
#ifndef OSB200_H_
#define OSB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum osb_status {
  OSB_OK = 0,
  OSB_ERR_INVALID = -1,   /* bad argument (shape, alignment, null pointer) */
  OSB_ERR_CUDA = -2,      /* CUDA runtime / driver error, see osb_last_error() */
  OSB_ERR_UNSUPPORTED = -3,
  OSB_ERR_NOT_INIT = -4
} osb_status;

/* ---- library management ------------------------------------------------------------------ */

/* Bind to `device`, resolve cuTensorMapEncodeTiled through the runtime, opt kernels into
 * large dynamic shared memory.  Must be called once per process and device before any op.
 * Fails with OSB_ERR_UNSUPPORTED on anything that is not compute capability 9.0. */
int osb_init(int device);
int osb_version(void);
const char* osb_last_error(void);
/* number of kernels this library has launched since process start (bench.py's gpu_launches) */
int64_t osb_launch_count(void);
/* hits / misses of the per-process TMA descriptor cache (descriptors are keyed by pointer, shape, stride and box) */
void osb_tmap_cache_stats(int64_t* hits, int64_t* misses);

/* ---- LayerNorm (no affine) + adaLN modulate ---------------------------------------------- */
/* y[r,:] = LN(x[r,:]) * (1 + scale[g,:]) + shift[g,:],  g = mod_index ? mod_index[r / group_rows]
 *                                                                     : r / group_rows
 * x,y: bf16 [rows, C] contiguous.  shift/scale: fp32, row g at shift + g*mod_stride (elements).
 * fp32 statistics (two-pass on register-resident row), eps as given (reference: 1e-6).
 * Replaces: opensora/models/mmdit/layers.py:205-206,223-224,248,252,312,400 (LayerNorm(no affine)
 * followed by (1+scale)*x+shift) and upstream v1.2 STDiT3 t2i_modulate(norm(x), shift, scale)
 * (SURVEY.md §8a-S).  C % 8 == 0, C <= 8192. */
int osb_ln_modulate(const void* x, const float* shift, const float* scale, void* y,
                    int64_t rows, int C, int64_t group_rows, const int32_t* mod_index,
                    int64_t mod_stride, float eps, void* stream);

/* ---- bf16 GEMM on wgmma with fused epilogues ---------------------------------------------- */
typedef enum osb_epilogue {
  OSB_EPI_BIAS = 0,           /* D = A W^T + bias                                              */
  OSB_EPI_BIAS_GELU_TANH = 1, /* D = gelu_tanh(A W^T + bias)      layers.py:277-281 (MLP[0:2]) */
  OSB_EPI_BIAS_GATE_RES = 2,  /* D = R + gate[g,:] * (A W^T + bias); gate==NULL -> plain add   */
                              /*                      layers.py:247-252, 333-334               */
  OSB_EPI_GATED_GELU = 3,     /* D[:, c] = gelu_tanh(P[:, 2c]) * P[:, 2c+1], P = A W^T + bias: W's rows interleave
                                 T5's wi_0 (even) and wi_1 (odd), D has N/2 columns (T5DenseGatedActDense)      */
  OSB_EPI_BIAS_QUICK_GELU = 4, /* D = x * sigmoid(1.702 x), x = A W^T + bias (CLIP mlp.fc1 + quick_gelu)         */
  OSB_EPI_BIAS_GELU_TANH_FP8 = 5 /* osb_gemm_fp8_blocks only: gelu_tanh(...) emitted as e4m3 with 1 x 128 block scales */
} osb_epilogue;

typedef struct osb_gemm_args {
  const void* A;       /* bf16 [M,K], row stride lda                                            */
  const void* W;       /* bf16 [N,K], row stride ldw  (nn.Linear.weight layout)                  */
  const void* bias;    /* bf16 [N] or NULL                                                       */
  void* D;             /* bf16 [M,N], row stride ldd                                             */
  const void* R;       /* bf16 [M,N] residual (GATE_RES only), row stride ldr; may alias D       */
  const float* gate;   /* fp32, row g at gate + g*gate_stride (GATE_RES only) or NULL            */
  const int32_t* mod_index; /* optional indirection for g, as in osb_ln_modulate                 */
  int64_t M, N, K;
  int64_t lda, ldw, ldd, ldr;
  int64_t group_rows;  /* g = row / group_rows                                                   */
  int64_t gate_stride;
  int32_t epilogue;    /* osb_epilogue                                                           */
  int32_t cta_group;   /* 0, 1 or 2; kept for ABI compatibility: sm_90a has no CTA-pair MMA, all run one CTA per tile */
  int32_t block_n;     /* 0 = library default, else 64/128/192/256                               */
  int32_t reserved;
} osb_gemm_args;

/* Replaces every nn.Linear on the block path: layers.py:209,212-214 (qkv / q,k,v proj),
 * :247,251 (attn out proj + gated residual), :277-281 (MLP), :314-333 (linear1/linear2), :401.
 * fp32 accumulation in registers; epilogue math in fp32; single rounding to bf16 on store.
 * Requires K % 8 == 0, N % 8 == 0. */
int osb_gemm_bf16(const osb_gemm_args* args, void* stream);

/* ---- LoRA: unmerged low-rank update in the same accumulator ------------------------------------------------------ */
typedef struct osb_lora_args {
  const void* U;  /* bf16 [M, r], row stride ldu: x · A^T (the down projection)          */
  const void* B;  /* bf16 [N, r], row stride ldb: scaling · lora_B                       */
  int64_t ldu, ldb;
  int32_t r;      /* multiple of 8 (the host zero-pads smaller ranks)                    */
  int32_t reserved;
  const float* col_scale; /* NULL, or fp32 [N], 8-byte aligned: DoRA's per-output-channel factor g */
} osb_lora_args;

/* D = epilogue(col_scale[n] * (A W^T + U B^T) + bias): osb_gemm_bf16 whose K loop is followed by ceil(r / 64) k-blocks
 * of U and B through the same wgmma pipeline, so the base product and the adapter's update share one fp32 accumulator
 * and one rounding to bf16 (merging the update into bf16 weights would round most of a small update away).  Every
 * epilogue, block_n and alignment rule of osb_gemm_bf16 applies.  The down projection U = x A^T is osb_gemm_bf16 with
 * N = r.  Replaces the unmerged peft LoRA layer the reference wraps the denoiser with (opensora/utils/sampling.py:542-545).
 *
 * col_scale (DoRA, weight-decomposed LoRA) multiplies the fp32 accumulator in registers, before the bias, GELU-tanh and
 * the gate / residual / mod_index rules; NULL means no scale.  It replaces peft's DoRA forward (peft/tuners/lora/dora.py,
 * DoraLinearLayer.forward at inference, dropout the identity):
 *     weight_norm    = || W + scaling * (lora_B @ lora_A) ||_2 per output row
 *     mag_norm_scale = lora_magnitude_vector / weight_norm
 *     result         = base(x) + (mag_norm_scale - 1) * x W^T + mag_norm_scale * scaling * lora_B(lora_A(x))
 * which equals g * (x W^T + scaling x A^T B^T) + bias with g = mag_norm_scale: the host computes g once per adapter and
 * passes it here.  An all-ones col_scale gives the bits of col_scale == NULL (x * 1.0f is exact). */
int osb_gemm_lora(const osb_gemm_args* gemm, const osb_lora_args* lora, void* stream);

/* ---- FP8 (e4m3) with per-row scales: the opt-in MLP path of STDiT3 ------------------------------------------------ */
/* Quantization rule shared by the three entry points below: a row r of a matrix X gets s[r] = amax(|X[r, :]|) / 448
 * (s = 1 for an all-zero row) and codes e4m3_rn_satfinite(X[r, k] / s[r]).  e4m3 tensors are one byte per element,
 * row-major with an explicit leading dimension in elements (= bytes). */
typedef struct osb_gemm_fp8_args {
  const void* A;         /* e4m3 [M,K], row stride lda                                                 */
  const void* W;         /* e4m3 [N,K], row stride ldw  (quantized nn.Linear.weight)                    */
  const float* a_scale;  /* fp32 [M]: the row scales of A                                               */
  const float* w_scale;  /* fp32 [N]: the row scales of W (per output channel)                          */
  const void* bias;      /* bf16 [N] or NULL                                                            */
  void* D;               /* bf16 [M,N], row stride ldd                                                  */
  const void* R;         /* bf16 [M,N] residual (GATE_RES only), row stride ldr; may alias D            */
  const float* gate;     /* fp32, row g at gate + g*gate_stride (GATE_RES only) or NULL                 */
  const int32_t* mod_index; /* optional indirection for g, as in osb_ln_modulate                       */
  int64_t M, N, K;
  int64_t lda, ldw, ldd, ldr;
  int64_t group_rows;    /* g = row / group_rows                                                        */
  int64_t gate_stride;
  int32_t epilogue;      /* OSB_EPI_BIAS, OSB_EPI_BIAS_GELU_TANH or OSB_EPI_BIAS_GATE_RES               */
  int32_t block_n;       /* 0 = library default, else 64 or 128                                         */
} osb_gemm_fp8_args;

/* D = epilogue(acc * (a_scale[m] * w_scale[n]) + bias), acc = the sum of the e4m3 products of row m of A and row n of W:
 * the tensor core (wgmma m64nNk32 e4m3) sums each 128-element k-block, whose partial is then added into an fp32
 * register accumulator (the FP8 MMA's own accumulation keeps fewer mantissa bits than fp32 and is never carried across
 * k-blocks).  The epilogues and their gate / residual / mod_index rules are those of osb_gemm_bf16, with one rounding
 * to bf16.  Replaces the two Linear layers of the STDiT3 block MLP when FP8 is enabled.
 * Requires K % 128 == 0, N % 8 == 0, lda, ldw multiples of 16 and 16-byte aligned A, W. */
int osb_gemm_fp8(const osb_gemm_fp8_args* args, void* stream);

/* osb_ln_modulate whose fp32 result row is quantized directly (no bf16 rounding) to e4m3 y8 [rows, C] (contiguous)
 * with its scale in y_scale[row].  Same group_rows / mod_index / mod_stride / eps arguments; C % 8 == 0, C <= 4096. */
int osb_ln_modulate_fp8(const void* x, const float* shift, const float* scale, void* y8, float* y_scale,
                        int64_t rows, int C, int64_t group_rows, const int32_t* mod_index,
                        int64_t mod_stride, float eps, void* stream);

/* Row quantizer: bf16 x [rows, K] (row stride ldx) -> e4m3 y8 [rows, K] (row stride ldy) and fp32 y_scale [rows], in
 * one pass over x (the row stays in registers between its amax and its codes).  K % 8 == 0, K <= 8192, ldx % 8 == 0,
 * ldy % 16 == 0, 16-byte aligned x and y8. */
int osb_quant_rows_fp8(const void* x, int64_t ldx, void* y8, int64_t ldy, float* y_scale, int64_t rows, int K,
                       void* stream);

/* ---- FP8 (e4m3) with 1 x 128 block scales: the opt-in MLP path of MMDiT -------------------------------------------- */
/* Block quantization rule: the block (r, b) = X[r, 128 b .. 128 b + 127] gets s[r, b] = amax(|block|) / 448 (s = 1 for an
 * all-zero block) and codes e4m3_rn_satfinite(X[r, k] / s[r, b]): the per-row rule applied per 128 columns. */
typedef struct osb_fp8_blocks_args {
  int64_t a_scale_ld;  /* 0: a_scale is fp32 [M] (per row); > 0: block mode, a_scale is fp32 [M, K/128] with this row
                          stride (>= K / 128)                                                                        */
  void* D8;            /* OSB_EPI_BIAS_GELU_TANH_FP8 only: e4m3 [M, N] codes, row stride ldd8 (D is not written)       */
  float* d_scale;      /* OSB_EPI_BIAS_GELU_TANH_FP8 only: fp32 [M, N/128] block scales, row stride ld_dscale          */
  int64_t ldd8, ld_dscale;
} osb_fp8_blocks_args;

/* osb_gemm_fp8 with the scales of A per (row, 128-element k-block): D = epilogue(w_scale[n] * sum_kb a_scale[m, kb] *
 * acc_kb + bias), acc_kb = the tensor core's sum over k-block kb, multiplied by its scale as it is promoted into the fp32
 * register accumulator.  Every epilogue of osb_gemm_fp8 (bias, GELU-tanh, gate + residual with group_rows / mod_index)
 * works in block mode.  a_scale_ld == 0 (per-row scales) with one of those epilogues runs osb_gemm_fp8 itself (same
 * kernel, same bits).
 * OSB_EPI_BIAS_GELU_TANH_FP8 (per-row or block-scaled A): v = gelu_tanh(acc * scales + bias) in fp32, written as e4m3
 * codes to D8 with one scale per (row, 128 columns) in d_scale, by the block quantization rule; no bf16 output.  Needs
 * N % 128 == 0 and block_n 0 or 128 (one output tile row = one scale block).  With D8 / d_scale pointing into the
 * columns of a wider buffer, it fills part of the A operand of a later block-mode GEMM.  Replaces fc1 -> GELU (and the
 * mlp part of linear1 -> GELU) of the MMDiT blocks when FP8 is enabled; block mode replaces fc2 and linear2. */
int osb_gemm_fp8_blocks(const osb_gemm_fp8_args* gemm, const osb_fp8_blocks_args* blk, void* stream);

/* osb_gemm_fp8_blocks plus an unmerged LoRA / DoRA update (osb_lora_args, as in osb_gemm_lora):
 *     D = epilogue(col_scale[n] * (w_scale[n] * sum_kb a_scale[m, kb] * acc_kb + sum_j U[m, j] * B[n, j]) + bias)
 * After the e4m3 k-blocks, ceil(r / 64) bf16 k-blocks of U [M, r] and B = scaling * lora_B [N, r] run through the same
 * pipeline; their partials are promoted into the same fp32 register accumulator unscaled, after w_scale has been applied
 * to the FP8 sum (w_scale never scales the update), and the one rounding is the epilogue's.  col_scale == NULL means 1;
 * an all-ones col_scale gives the bits of NULL.  Every epilogue of osb_gemm_fp8_blocks works, per-row (a_scale_ld == 0)
 * or block-scaled A: bias, GELU-tanh, gate + residual (group_rows / mod_index, R may alias D) and, with block_n 0 or
 * 128, OSB_EPI_BIAS_GELU_TANH_FP8, where the update enters before the GELU and the block amax.
 * The down projection U = x A_cat^T is osb_gemm_fp8_blocks with N = r on the same e4m3 input (A_cat quantized per row
 * by osb_quant_blocks_fp8 with block = K) and a bf16 output.
 * Requirements: those of osb_gemm_fp8_blocks, plus those of osb_gemm_lora: r > 0 and r % 8 == 0, U and B 16-byte
 * aligned with ldu, ldb >= r and multiples of 8, col_scale 8-byte aligned.
 * Returns OSB_ERR_INVALID for a null gemm, blk or lora argument, a null operand or scale, any shape, stride or alignment
 * rule above, or an epilogue it does not build; OSB_ERR_UNSUPPORTED for block_n other than 0, 64 or 128;
 * OSB_ERR_NOT_INIT before osb_init().  Runs the adapted block Linears of MMDiT when FP8 is enabled with lora=True. */
int osb_gemm_fp8_lora(const osb_gemm_fp8_args* gemm, const osb_fp8_blocks_args* blk, const osb_lora_args* lora,
                      void* stream);

/* Block quantizer: bf16 x [rows, K] (row stride ldx) -> e4m3 y8 [rows, K] (row stride ldy) with the scale of (row r,
 * block b) at y_scale[r * lds + b].  block == 128: 1 x 128 block scales, one pass over x (the attention output of the
 * MMDiT single blocks).  block == K: one scale per row for rows of any length (the MLP weights, per output channel, up
 * to K = 5 x 4096; the row is read twice).  K % 128 == 0, ldx and ldy multiples of 8, 16-byte aligned x, 8-byte aligned
 * y8, 4-byte aligned y_scale. */
int osb_quant_blocks_fp8(const void* x, int64_t ldx, void* y8, int64_t ldy, float* y_scale, int64_t lds, int64_t rows,
                         int K, int block, void* stream);

/* ---- FP8 (e4m3) attention: the opt-in attention path of MMDiT -------------------------------------------------------- */
/* Self-attention of the joint txt|img sequence of MMDiT on e4m3 operands.  Inputs are described by osb_attn_short_args
 * with head_dim == 128, Lq == Lk == L (any L >= 1), seqs_per_batch == 1, kv_lens == NULL, any number of heads.  Per
 * sequence b, head h (bh = b * num_heads + h) and token t:
 *   q, k:  q~ = the bf16 row osb_attn_short stages (RMSNorm with the weight of the token's stream, RoPE, one rounding);
 *          s_q[bh, t] = amax(|q~|) / 448 (1 for a zero row), codes e4m3_rn_satfinite(q~ / s_q): the per-row rule of the
 *          FP8 GEMMs applied per (token, head).  k likewise.
 *   v:     one scale per channel over the sequence: s_v[bh, c] = amax_t(|v[t, c]|) / 448 (1 for a zero column), codes
 *          e4m3_rn_satfinite(v / s_v).
 *   scores (log2 units, fp32):  S_ij = s_q[i] * s_k[j] * (sum_d q8[i, d] k8[j, d]) * softmax_scale * log2(e).
 *   softmax: online over key blocks of 128, p = exp2(S - m_running) in fp32, l = fp32 sum of p.
 *   PV:    P8 = e4m3_rn_satfinite(256 * p) (2^8: p down to ~2^-17 keeps a nonzero code, nothing saturates); each key
 *          block's P8 V8 is summed by the tensor core into a partial that is promoted into the fp32 accumulator as
 *          O = alpha * O + partial (the FP8 MMA accumulates with fewer mantissa bits than fp32).
 *   out[row of (b, i), h * 128 + c] = bf16(O_ic * s_v[c] / (256 * l_i)), rows and columns as osb_attn_short writes them.
 *
 * Workspace (caller-owned, device memory; Lpad = L rounded up to a multiple of 128, the key block):
 *   q8, k8   e4m3 [B*H, Lpad, 128], rows t >= L hold zero codes with scale 1
 *   vt8      e4m3 [B*H, 128, Lpad]: V transposed (keys contiguous: FP8 wgmma reads B K-major only), and within every group
 *            of 32 keys g*32 + j the key at position p is j(p) = 16*(p/16) + 2*((p%16)/4) + (p%2) + 8*((p%4)/2), so that
 *            the S accumulator registers of a thread are the register A fragment of the PV product as they are; pad keys
 *            hold zero codes
 *   s_q, s_k fp32 [B*H, Lpad]
 *   s_v      fp32 [B*H, 128]
 *   v_amax   fp32 [B*H, 128] scratch: must be all zero before the first call (each call leaves it zero again, on the
 *            stream, so the path has no host synchronisation and is graph-capturable)
 * All pointers 16-byte aligned; capacity_bh >= B*H and capacity_lpad >= Lpad describe the buffers' extents, and the
 * strides above are those of the CALL's Lpad (the buffers are viewed densely for each call). */
typedef struct osb_attn_fp8_workspace {
  void* q8; void* k8; void* vt8;
  float* s_q; float* s_k; float* s_v;
  float* v_amax;
  int64_t capacity_bh, capacity_lpad;
} osb_attn_fp8_workspace;

/* Three launches: prep (q / k quantized rows with their scales, v's channel amax by atomicMax on the non-negative
 * float bits), V pack (scales, transposed permuted codes), attention (wgmma e4m3 x e4m3 -> fp32, TMA-fed).  Refuses
 * head_dim != 128, Lq != Lk, kv_lens, seqs_per_batch != 1, misaligned pointers and a workspace too small. */
struct osb_attn_short_args;   /* defined with osb_attn_short below */
int osb_attn_fp8(const struct osb_attn_short_args* args, const osb_attn_fp8_workspace* ws, void* stream);

/* Block-scaled e4m3 output of osb_attn_fp8.  With head_dim 128 one (row, head) of the output is one 1 x 128 block of
 * the block quantization rule (osb_fp8_blocks_args): v = O_ic * s_v[c] / (256 * l_i) in fp32 (the value osb_attn_fp8
 * rounds to bf16), s = amax_c(|v|) / 448 (1 for an all-zero block), codes e4m3_rn_satfinite(v / s) (IEEE division).
 * Rows follow the row mapping of args->out:
 *   codes   e4m3, element (row, h * 128 + c) at codes + row * codes_ld + h * 128 + c
 *   scales  fp32, the scale of (row, h) at scales[row * scales_ld + h]
 * With codes / scales pointing into the columns of a wider buffer the output fills part of the block-scaled A operand
 * of osb_gemm_fp8_blocks (the attention half of linear2's input, or the input of an attention-output projection). */
typedef struct osb_attn_fp8_out {
  void* codes;       /* 16-byte aligned, codes_ld a multiple of 8           */
  float* scales;     /* 4-byte aligned, scales_ld >= num_heads              */
  int64_t codes_ld, scales_ld;
} osb_attn_fp8_out;

/* osb_attn_fp8 writing `out` instead of args->out (which is not read): the same three launches, workspace and refusals;
 * the attention kernel quantizes in its epilogue. */
int osb_attn_fp8_blocks(const struct osb_attn_short_args* args, const osb_attn_fp8_workspace* ws,
                        const osb_attn_fp8_out* out, void* stream);

/* ---- attention with short key sets (whole key set resident in one CTA) -------------------- */
typedef struct osb_attn_short_args {
  const void* q; const void* k; const void* v; /* bf16; element (row, h*D + d) at ptr + row*ld + h*D + d */
  void* out;                                   /* bf16 [*, out_ld], same row mapping as q        */
  int64_t q_ld, k_ld, v_ld, out_ld;
  /* row mapping: sequence s -> (b = s / seqs_per_batch, j = s % seqs_per_batch);
   * q row of token t = b*q_batch_stride + j*q_seq_stride + t*q_tok_stride  (same for k/v with k_*) */
  int64_t num_seqs, seqs_per_batch;
  int64_t q_batch_stride, q_seq_stride, q_tok_stride;
  int64_t k_batch_stride, k_seq_stride, k_tok_stride;
  int32_t Lq, Lk;                 /* tokens per sequence (Lq < 128: 128 / Lq sequences share a query tile) */
  const int32_t* kv_lens;         /* optional [num_seqs]: valid keys per sequence (<= Lk)       */
  int32_t num_heads, head_dim;    /* head_dim: 72 (STDiT3-XL) or 64                              */
  const void* q_norm_w;           /* bf16 [D] RMSNorm weight for q, or NULL = no QK-norm         */
  const void* k_norm_w;           /* bf16 [D]                                                    */
  float norm_eps;
  const float* rope_cos;          /* fp32 [Lmax, D/2] or NULL: interleaved-pair RoPE by token    */
  const float* rope_sin;          /*   index (rotary_embedding_torch layout, SURVEY App. A)      */
  float softmax_scale;            /* D^-0.5                                                      */
  const void* q_norm_w2;          /* optional second RMSNorm weight pair used by tokens >= norm_split: the     */
  const void* k_norm_w2;          /*   joint txt|img sequence of MMDiT has per-stream QKNorm (layers.py:222,238) */
  int32_t norm_split;
  int32_t reserved;               /* implementation switch, kept for ABI compatibility: every value runs the one
                                     flash-attention kernel of sm_90a */
  int32_t rope_half;              /* 1: rope tables are applied with the rotate-half pairing (i, i + D/2) of HF /   */
  int32_t reserved2;              /*    Liger RoPE (math.py:27); 0: interleaved pairs (2i, 2i+1) (math.py:60-65)     */
} osb_attn_short_args;

/* softmax(q k^T * scale) v per (sequence, head), non-causal, optional per-head RMSNorm on q,k
 * and RoPE applied while staging operands into shared memory.  A row with no valid key (kv_lens
 * 0) is written as zeros.  Replaces: mmdit/math.py:22-36
 * (`attention`), layers.py:126-135 (QKNorm), and upstream STDiT3 Attention / MultiHeadCrossAttention
 * (SURVEY.md §8a-S, Appendix A). */
int osb_attn_short(const osb_attn_short_args* args, void* stream);

/* osb_attn_short with an additive fp32 bias by relative position: the score of query token i and key token j is
 * q.k * softmax_scale + bias[h * bias_head_stride + j - i + Lq - 1] (bias: [heads][Lq + Lk - 1], or one shared vector
 * with bias_head_stride = 0), added before the running maximum.  -inf entries mask keys; key blocks that are -inf for
 * every query of a 128-row query tile are skipped, and a row never evaluates -inf - (-inf): a row whose every key is
 * masked is written as zeros.  head_dim 64 only; kv_lens and packed short sequences as in osb_attn_short; QK-norm and
 * RoPE arguments keep their meaning.
 * Replaces the self-attention of HF T5Attention (relative_attention_bias, unscaled scores: softmax_scale = 1) and
 * CLIPAttention (causal mask: bias 0 for j <= i, -inf for j > i) run by the reference's text_embedder
 * (opensora/models/text/conditioner.py:10-53). */
int osb_attn_short_bias(const osb_attn_short_args* args, const float* bias, int64_t bias_head_stride, void* stream);

/* ---- frame-causal attention of one 512-wide head (causal VAE mid block) ---------------------------------------------- */
typedef struct osb_attn_frames_args {
  const void* q; const void* k; const void* v;   /* bf16; element (row, d) at ptr + row * ld + d, d < 512            */
  void* out;                                     /* bf16, rows mapped like q                                        */
  int64_t q_ld, k_ld, v_ld, out_ld;              /* >= 512, multiples of 8 (q | k | v may be slices of one buffer)  */
  int64_t q_batch_stride, k_batch_stride;        /* rows between samples (out uses q's, v uses k's)                 */
  int64_t Lq, Lk;                                /* query / key tokens per sample                                   */
  int32_t batch, head_dim;                       /* head_dim: 512, anything else is refused                         */
  int32_t frame_tokens;                          /* hw: tokens per latent frame, any value >= 1                     */
  int32_t q_frame0;                              /* global frame of query token 0 (frame-sharded VAE: `first`)      */
  float softmax_scale;                           /* 512^-0.5                                                        */
  int32_t reserved;
} osb_attn_frames_args;

/* out = softmax(q k^T * softmax_scale + frame mask) v for ONE head of 512 channels.  Query token i of a sample sees key
 * j iff j < min(Lk, (q_frame0 + i / frame_tokens + 1) * frame_tokens): the mask of `prepare_causal_attention_mask` as a
 * predicate, never a tensor; key blocks past a query tile's last visible key are not read.  With Lk > Lq and q_frame0 > 0
 * the queries are a run of frames of a longer video whose keys / values were gathered (frame-sharded VAE).
 * Arithmetic: scores in fp32 in log2 units, exact online softmax over 128-key blocks with a guarded running maximum,
 * P rounded to bf16 unnormalised, O accumulated and rescaled in fp32, one rounding at the output.  Deterministic (no
 * atomics, keys are never split across CTAs).  One CTA per 64 query rows: wgmma for both products, q / k / v loaded by TMA
 * as they lie in memory (v is never transposed).
 * Refused before any launch: head_dim != 512, an ld below 512 or not a multiple of 8, pointers not 16-byte aligned,
 * frame_tokens < 1, batch < 1, Lq < 1, batch strides that are negative or shorter than the sample, softmax_scale <= 0,
 * and q_frame0 < 0 or Lk < 1 (some query would see no key).
 * Replaces the mid-block attention of the reference's causal VAE: the mask of
 * opensora/models/hunyuan_vae/unet_causal_3d_blocks.py:52-60, the one-head Attention built at :311-325 and its call at
 * :349-352 (diffusers' AttnProcessor2_0 -> scaled_dot_product_attention with that mask). */
int osb_attn_frames(const osb_attn_frames_args* args, void* stream);

/* ---- RMSNorm with weight (T5LayerNorm) ----------------------------------------------------------------------------- */
/* y[r,:] = bf16(w * bf16(x[r,:] * rsqrt(mean(x[r,:]^2) + eps))): fp32 mean of squares, the reference's two roundings
 * (opensora/acceleration/shardformer/modeling/t5.py:14-27).  x, y: bf16 [rows, C] contiguous, w: bf16 [C].
 * C % 8 == 0, C <= 4096 (T5-XXL's d_model), 16-byte aligned.  One warp per row, one HBM pass. */
int osb_rms_norm(const void* x, const void* w, void* y, int64_t rows, int C, float eps, void* stream);

/* ---- head tiles: projection GEMM -> attention without a layout pass ------------------------------------ */
/* A head tile is the HBM image of one attention operand tile: tile_rows <= 128 token rows of ONE head, head_dim
 * padded to a multiple of 16, 64-column chunks in the 128-byte-swizzle layout followed by the head-dim tail in the
 * no-swizzle core-matrix layout (open-sora_b200/csrc/tiles.cuh).  The projection GEMM writes q / k / v straight into
 * this form (bias + per-head RMSNorm + RoPE fused in its epilogue) and the attention kernel loads whole tiles with
 * one bulk copy each.  osb_tile_map says which token row lands in which (tile, row):
 *   mode 0: sequences are contiguous row blocks        seq = row / L, pos = row % L
 *   mode 1: frame-major stream viewed along T          row = (b*T + t)*S + s -> seq = b*S + s, pos = t  (L == T)
 *   G > 1 : G short sequences packed per tile          tile = seq / G, r = (seq % G)*L + pos   (G*L <= tile_rows, tps == 1)
 *   G == 1: tile = seq*tps + pos / tile_rows, r = pos % tile_rows, tps = ceil(L / tile_rows)                      */
struct osb_scatter;
typedef struct osb_tile_map {
  int32_t mode, L, S, T, G, tps, tile_rows, reserved;
} osb_tile_map;

typedef struct osb_head_tiles_args {
  void* tiles;              /* tile buffer; tile (kidx, head, t) at tiles + kidx*kind_stride + head*head_stride +
                               t*tile_rows*2*pad16(head_dim), kidx = output column / (num_heads*head_dim)           */
  int64_t kind_stride;      /* bytes between consecutive num_heads*head_dim wide column groups (q | k | v, or the
                               k | v pairs of several blocks)                                                        */
  int64_t head_stride;      /* bytes between heads = tiles per head * tile bytes                                     */
  osb_tile_map map;
  int32_t num_heads, head_dim;
  int32_t nkinds;           /* column group kidx is of kind kidx % nkinds                                            */
  uint32_t norm_mask;       /* bit k: kind k gets per-head RMSNorm with norm_w[k]        (layers.py:102-135)         */
  uint32_t rope_mask;       /* bit k: kind k gets interleaved-pair RoPE by position      (math.py:60-65)             */
  int32_t reserved;         /* kept for ABI compatibility (bit 0 selected a store path that sm_90a does not have): the
                               epilogue stores every head row straight into its tile                                  */
  const void* norm_w[4];    /* bf16 [head_dim] per kind or NULL                                                      */
  float norm_eps;
  int32_t reserved2;
  const float* rope_cos;    /* fp32 [L, head_dim/2]                                                                  */
  const float* rope_sin;
} osb_head_tiles_args;

/* tiles = head_tiles(epilogue(A W^T + bias)): the GEMM of osb_gemm_bf16 (gemm->D / ldd / epilogue / R / gate are
 * ignored) whose epilogue splits every output row into heads, applies RMSNorm / RoPE in fp32 on the fp32
 * accumulator and stores each head row once, as bf16, at its place in the tile buffer.
 * Replaces layers.py:209-214 (qkv Linear), :116-135 (QKNorm) and math.py:27,60-65 (RoPE) - the q/k/v tensors in
 * token layout never exist.  Requires N % (num_heads*head_dim) == 0, head_dim in {64, 72, 128}. */
int osb_gemm_head_tiles(const osb_gemm_args* gemm, const osb_head_tiles_args* tiles, void* stream);

/* tiles per head for `rows` token rows under `map` (rows / L sequences) */
int64_t osb_head_tiles_per_head(const osb_tile_map* map, int64_t rows);

typedef struct osb_attn_tiles_args {
  const void* q_tiles; const void* k_tiles; const void* v_tiles;  /* tile 0 of head 0 of each operand                */
  int64_t q_head_stride, kv_head_stride;                          /* bytes between heads                            */
  osb_tile_map q_map;        /* rows of `out` <-> q tiles; key set i belongs to sequence i (G == 1) or tile i (G > 1).
                                The map may differ from the one the tiles were written with in `mode` only (tiles produced
                                from a transposed [B, S, T] stream with mode 0, output rows frame-major with mode 1)      */
  int32_t kv_tile_rows;      /* rows per key / value tile (multiple of 16, <= 128)                                  */
  int32_t kv_tiles_per_set;  /* key tiles per sequence: ceil(Lk / kv_tile_rows) (1 for packed sequences)            */
  int32_t Lk;                /* keys per sequence                                                                   */
  int32_t num_heads, head_dim;
  int32_t reserved;
  int64_t num_seqs;
  const int32_t* kv_lens;    /* optional [num_seqs]: valid keys per sequence (G == 1)                               */
                             /* With a packed q map (G > 1) kv_lens is not read: every packed sequence sees its Lk keys.
                                The Python binding refuses kv_lens with a packed map rather than ignore it.            */
  void* out;                 /* bf16, row of token = inverse of q_map, head h at columns [h*head_dim, (h+1)*head_dim) */
  int64_t out_ld;
  float softmax_scale;
  int32_t reserved2;
  const struct osb_scatter* out_scatter; /* optional: route output rows to peer buffers (sequence parallel), else NULL   */
} osb_attn_tiles_args;

/* out = softmax(q k^T * scale) v per (sequence, head) over head tiles: one CTA per (query tile, head), bulk-copy loads
 * with the next key tile in flight (open-sora_b200/csrc/attn_sm90.cu).  An empty key set (kv_lens 0) writes zeros.  Replaces mmdit/math.py:22-36. */
int osb_attn_tiles(const osb_attn_tiles_args* args, void* stream);

/* ---- FP8 (e4m3) head-tile attention: the opt-in attention path of STDiT3 ---------------------------------------------- */
/* The bf16 head tiles written by osb_gemm_head_tiles (bias, QK-RMSNorm and RoPE applied, rounded once) are converted to
 * e4m3 tiles, and osb_attn_tiles_fp8 computes every set shape of osb_attn_tiles on them.  head_dim 72 or 64 only.
 *   q, k:  one scale per (token, head): s = amax(|row|) / 448 (1 for an all-zero row), codes e4m3_rn_satfinite(row / s):
 *          the per-row rule of the FP8 GEMMs.
 *   v:     one scale per (key tile, head, channel) over the tile's rows, by the same rule.  A packed temporal tile
 *          shares one scale among its G short sequences; no reduction crosses tiles.
 *   scores (log2 units, fp32):  S_ij = s_q[i] * s_k[j] * (sum_d q8[i, d] k8[j, d]) * softmax_scale * log2(e).
 *   softmax: online over key tiles, p = exp2(S - m_running) in fp32, l = fp32 sum of p.
 *   PV:    P8 = e4m3_rn_satfinite(256 * p); each key tile's P8 V8 is summed by the tensor core into a partial promoted as
 *          O = alpha * O + s_v[tile] (.) partial (per channel).
 *   out = bf16(O / (256 * l)), rows addressed as osb_attn_tiles addresses them (inverse q_map, optional out_scatter).
 *   Masks: packed sequences (G > 1) are block-diagonal inside a tile, kv_lens applies when G == 1, the last tile may be
 *   ragged, and an empty key set writes zeros (as osb_attn_tiles does).
 *
 * Tile format (open-sora_b200/csrc/tiles.cuh): every tile is 128 rows x 128 bytes of e4m3 codes (16384 bytes) in the
 * 128-byte swizzle (byte c of row r at r * 128 + (((c / 16) ^ (r % 8)) * 16) + c % 16) plus 128 fp32 scales.
 *   q / k tile: row = tile row, byte = channel (channels >= head_dim and rows >= tile_rows: zero codes, scale 1).
 *   v tile:     row = channel (rows >= head_dim unused), byte p = key j(p) of the tile with the osb_attn_fp8 vt8 order
 *               j(p) = 32*(p/32) + 16*((p%32)/16) + 2*((p%16)/4) + (p%2) + 8*((p%4)/2); scales per channel (1 past
 *               head_dim).
 * Tile (kind, head, t) sits at index (kind * num_heads + head) * tiles_per_head + t of both arrays, t the tile index of
 * the bf16 buffer it came from. */
typedef struct osb_tiles_fp8 {
  void* codes;              /* e4m3, 16384 bytes per tile, 16-byte aligned                                           */
  float* scales;            /* fp32 [tiles][128], 16-byte aligned                                                    */
  int64_t tiles_per_head;
  int32_t num_heads, reserved;
} osb_tiles_fp8;

typedef struct osb_head_tiles_fp8_args {
  const void* tiles;        /* bf16 head tiles of the first kind converted (osb_head_tiles_args layout)              */
  int64_t kind_stride, head_stride;   /* bytes, as in osb_head_tiles_args                                            */
  osb_tiles_fp8 dst;        /* e4m3 tiles: dst tile (k, head, t) <- source tile (k, head, t), k < nkinds             */
  int32_t tile_rows, head_dim;
  int32_t nkinds;           /* kinds converted in this launch                                                        */
  int32_t v_period, v_slot; /* kind k is a value kind iff v_period > 0 and k % v_period == v_slot (q|k|v: 3, 2;
                               the k|v pairs of all blocks: 2, 1; queries only: 0, 0)                                */
  int32_t reserved;
} osb_head_tiles_fp8_args;

/* One launch, one CTA per (tile, head, kind): q / k tiles get per-row codes and scales, v tiles are transposed and
 * scaled per channel.  Any run of kinds converts in one launch (the text keys / values of all 2*depth blocks at once). */
int osb_head_tiles_fp8(const osb_head_tiles_fp8_args* args, void* stream);

typedef struct osb_attn_tiles_fp8_operands {
  const void* q8; const void* k8; const void* v8;     /* e4m3 tile 0 of head 0 of the q, k and v kinds               */
  const float* s_q; const float* s_k; const float* s_v; /* the scales of the same tiles                               */
  int64_t q_head_tiles, kv_head_tiles;                /* tiles between heads (tiles_per_head of each buffer)         */
} osb_attn_tiles_fp8_operands;

/* osb_attn_tiles on e4m3 tiles: every field of `args` keeps its meaning except q_tiles / k_tiles / v_tiles and the two
 * head strides, which are not read (`ops` gives the e4m3 tiles).  head_dim 72 or 64.  One CTA of three warpgroups per
 * (query tile, head): a producer streams K / V tiles and their scales with bulk copies through an mbarrier ring, two
 * consumers run S = Q K^T and P8 V8 on wgmma e4m3. */
int osb_attn_tiles_fp8(const osb_attn_tiles_args* args, const osb_attn_tiles_fp8_operands* ops, void* stream);

/* ---- sequence-parallel exchange over peer memory (NVLink / NVSwitch; SURVEY.md §8b, §8e) ------------------------- */
/* The T-shard <-> S-shard transposition around temporal attention (the reference's all_to_all,
 * opensora/acceleration/communications.py:8-18,57-63) is done by the PRODUCING kernel: it stores every output row
 * straight into the buffer of the rank that will consume it (peer-mapped symmetric memory created on the Python side,
 * torch.distributed._symmetric_memory), so there is no pack copy, no collective call and no unpack copy.  osb_scatter
 * describes the row routing; osb_comm_barrier is the one small kernel that orders producers and consumers across ranks.
 * NCCL itself stays in Python (torch.distributed) for the entry split / exit all-gather. */
#define OSB_MAX_PEERS 16
typedef struct osb_scatter {
  int32_t mode;   /* 0: none (plain local output).  Rows are viewed as [B, I, J]:
                     1: J is split over the P ranks: row (b, i, j) goes to rank p = j / (J/P), row
                        (b*(P*I) + rank*I + i) * (J/P) + j % (J/P) of its buffer   ([B, Tl, S] -> [B, T, S/P]);
                     2: I is split: row (b, i, j) goes to rank p = i / (I/P), row
                        (b*(I/P) + i % (I/P)) * (P*J) + rank*J + j of its buffer   ([B, T, Sl] -> [B, T/P, S]);
                     3: no exchange, rows transposed: (b, i, j) -> row (b*J + j)*I + i of peer[rank]
                        ([B, T, S] -> [B, S, T]: temporal sequences become contiguous row blocks for the QKV GEMM);
                     4: mode 1 with the destination transposed: rank p = j / (J/P) gets row
                        (b*(J/P) + j % (J/P)) * (P*I) + rank*I + i   ([B, Tl, S] -> [B, S/P, T])                     */
  int32_t P, rank, I, J;
  int32_t reserved[3];
  void* peer[OSB_MAX_PEERS];   /* base of the destination buffer on every rank (peer[rank] is the local one)           */
} osb_scatter;

/* osb_ln_modulate with the output rows routed by `scatter` (row stride C elements on every destination) */
int osb_ln_modulate_scatter(const void* x, const float* shift, const float* scale, int64_t rows, int C,
                            int64_t group_rows, const int32_t* mod_index, int64_t mod_stride, float eps,
                            const osb_scatter* scatter, void* stream);

typedef struct osb_comm_barrier_args {
  int32_t P, rank;
  uint32_t* epoch;                   /* local device counter: exchanges completed so far (the kernel increments it)    */
  uint32_t* flags_local;             /* [P] slots other ranks write into                                               */
  uint32_t* flags_peer[OSB_MAX_PEERS]; /* the same array on every rank, peer-mapped                                    */
} osb_comm_barrier_args;

/* One CTA: thread p publishes "my stores of exchange e are done" (st.release.sys) into slot `rank` of rank p's flags,
 * then waits (ld.acquire.sys) until slot p of the local flags reached e.  Stream order before it = this rank's producer
 * has completed; after it = every rank's producer has.  Capturable in a CUDA graph (the epoch lives on the device). */
int osb_comm_barrier(const osb_comm_barrier_args* args, void* stream);

/* ---- causal 3D VAE: implicit-GEMM convolution + its HBM-bound helpers ----------------------------- */
typedef struct osb_conv3d_args {
  const void* x_pad;    /* bf16 NDHWC [nb, tp, hp, wp, cp]: input ALREADY padded (replicate; T front only) by
                           osb_vae_prep; in narrow mode the buffer must extend 128 bytes past its end        */
  const void* w;        /* bf16 [cout, K] K-major.  normal: K = kt*kh*kw*cp, k = ((it*kh+ih)*kw+iw)*cp + c;
                           narrow: K = kt*kh*64, k = (it*kh+ih)*64 + iw*cp + c (zero where iw*cp+c >= kw*cp)  */
  const void* bias;     /* bf16 [cout] or NULL                                                                 */
  void* y;              /* bf16 NDHWC [nb, t_out, h_out, w_out, cout]                                          */
  const void* residual; /* bf16 like y, added in fp32 before the single rounding; or NULL                      */
  int32_t nb, tp, hp, wp, cp;
  int32_t t_out, h_out, w_out, cout;
  int32_t st, sh, sw;   /* strides (1 or 2)                                                                    */
  int32_t kt, kh, kw;   /* taps (1..3)                                                                         */
  int32_t narrow;       /* 1: cp in {8,16}, the kw taps x cp channels form one 64-element K block             */
  int32_t block_n;      /* 0 = library default                                                                 */
} osb_conv3d_args;

/* y = conv3d(x_pad) + bias (+ residual), fp32 accumulation in registers, one rounding to bf16.  Every k-block is a
 * 5-D TMA box load of the padded NDHWC input at the tap offset (strided boxes for stride-2 convolutions), fed to
 * the same wgmma main loop and epilogue as osb_gemm_bf16.
 * Replaces: opensora/models/hunyuan_vae/unet_causal_3d_blocks.py:94-96 (CausalConv3d.forward: F.pad replicate +
 * ChannelChunkConv3d) and opensora/models/vae/utils.py:172-190 (the cuDNN conv3d it dispatches to). */
int osb_conv3d_ndhwc(const osb_conv3d_args* args, void* stream);

/* GroupNorm statistics over an NDHWC tensor: for every (n, group) the mean and 1/sqrt(var + eps) over
 * (C/groups) channels x T*H*W positions -> mean_rstd fp32 [nb, groups, 2].  Deterministic (no atomics): fp32
 * partials per 2048-position chunk in `workspace` (osb_group_stats_workspace_bytes), fixed-order fp64 finalisation.
 * Replaces the statistics half of torch.nn.GroupNorm at unet_causal_3d_blocks.py:216,218,246-250; vae.py:115,229. */
int64_t osb_group_stats_workspace_bytes(int64_t nb, int64_t positions, int32_t groups);
int osb_group_stats(const void* x, int64_t nb, int64_t positions, int32_t C, int32_t groups, float eps,
                    void* workspace, int64_t workspace_bytes, float* mean_rstd, void* stream);

typedef struct osb_vae_prep_args {
  const void* x;           /* bf16 NDHWC [nb, t, h, w, c]                                                      */
  void* y;                 /* bf16 NDHWC [nb, tp, hp, wp, cp]                                                  */
  const float* mean_rstd;  /* [nb, groups, 2] from osb_group_stats, or NULL = no normalisation                 */
  const void* gamma;       /* bf16 [c] GroupNorm weight (with mean_rstd)                                       */
  const void* beta;        /* bf16 [c]                                                                         */
  int32_t nb, t, h, w, c;
  int32_t groups;
  int32_t silu;            /* apply x*sigmoid(x) after the affine                                              */
  int32_t ft, fh, fw;      /* nearest-neighbour upsample factors (1 or 2); T rule: frame 0 -> 1 frame, others x ft */
  int32_t pad_t, pad_h, pad_w; /* replicate padding: pad_t frames in FRONT only, pad_h / pad_w on both sides    */
  int32_t cp;              /* output channels >= c (zero filled), multiple of 8                                */
} osb_vae_prep_args;

/* One HBM pass that produces the convolution's input: GroupNorm apply + SiLU + nearest upsample (first-frame
 * rule) + replicate padding, written channels-last.  Replaces the separate GroupNorm / SiLU / F.interpolate /
 * F.pad passes of unet_causal_3d_blocks.py:95,136-150,246-250. */
int osb_vae_prep(const osb_vae_prep_args* args, void* stream);

/* ---- sampler step (SURVEY.md §8f-1) --------------------------------------------------------------------- */
/* pred = uncond2 + g_img*(uncond - uncond2) + g_txt*(cond - uncond)  (uncond2 == NULL: uncond + g_txt*(cond - uncond));
 * out = x + dt*pred.  bf16 [n] in/out (out may alias x), fp32 math, one rounding.  g_img_map: optional bf16 map of
 * per-element image guidance repeating with period map_period (temporal oscillation).
 * Replaces opensora/utils/sampling.py:204-222 (CFG combine + Euler update of I2VDenoiser.denoise). */
int osb_cfg_euler(const void* cond, const void* uncond, const void* uncond2, const void* x, void* out, int64_t n,
                  float g_txt, float g_img, const void* g_img_map, int64_t map_period, float dt, void* stream);

/* Frame-masked step of image / video conditioning (Open-Sora v1.2 RFLOW.sample, mask branch; parity unpinned): the end
 * of sampling step i fused with the start of step i + 1, in one pass over x.  N = num_timesteps; per frame (b, f) with
 * m = frame_mask[b, f] * N (1 = generate, 0 = keep the reference, in between = edit ratio):
 *   update:  m >= t_cur[b]  -> x' = x + dt * (uncond + guidance * (cond - uncond)),  dt = (t_cur[b] - t_next[b]) * (1/N)
 *            (the fp32 expression of osb_cfg_euler's two-branch mode, and dt as torch computes (t_cur - t_next) / N on
 *            the GPU: an all-ones mask gives the bits of osb_cfg_euler called with that dt);
 *            otherwise x' = x, bit for bit.  update == 0 (prologue, launched once before the first model call): x' = x.
 *   re-noise (noise != NULL): prev = update ? (m >= t_cur[b]) : (frame_mask[b, f] == 1);
 *            m >= t_next[b] && !prev -> out = (1 - a) * x' + a * noise, a = t_next[b] * (1/N);  otherwise out = x'.
 * cond, uncond, x, noise, out: bf16 [B, C, T, H*W] contiguous, 16-byte aligned; out may alias x.  cond / uncond may be
 * NULL when update == 0; noise may be NULL when update != 0.  frame_mask: fp32 [B, T]; t_cur, t_next: DEVICE fp32 [B]
 * (per-sample schedules in one launch, no host synchronisation: the call is graph-capturable and a replay reads the
 * current contents).  fp32 math, one rounding per element.  Any H*W (16-byte vectors when H*W % 8 == 0).
 * Replaces the torch add_noise / where / CFG / Euler ops of each step of v1.2 schedulers/rf/__init__.py::RFLOW.sample. */
int osb_rf_masked_step(const void* cond, const void* uncond, const void* x, const void* noise, void* out,
                       const float* frame_mask, const float* t_cur, const float* t_next, int32_t B, int32_t C, int32_t T,
                       int64_t HW, float guidance, int32_t num_timesteps, int32_t update, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OSB200_H_ */
