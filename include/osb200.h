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
  OSB_EPI_BIAS_QUICK_GELU = 4 /* D = x * sigmoid(1.702 x), x = A W^T + bias (CLIP mlp.fc1 + quick_gelu)          */
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
} osb_lora_args;

/* D = epilogue(A W^T + U B^T + bias): osb_gemm_bf16 whose K loop is followed by ceil(r / 64) k-blocks of U and B
 * through the same wgmma pipeline, so the base product and the adapter's update share one fp32 accumulator and one
 * rounding to bf16 (merging the update into bf16 weights would round most of a small update away).  Every epilogue,
 * block_n and alignment rule of osb_gemm_bf16 applies.  The down projection U = x A^T is osb_gemm_bf16 with N = r.
 * Replaces the unmerged peft LoRA layer the reference wraps the denoiser with (opensora/utils/sampling.py:542-545). */
int osb_gemm_lora(const osb_gemm_args* gemm, const osb_lora_args* lora, void* stream);

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
 * and RoPE applied while staging operands into shared memory.  Replaces: mmdit/math.py:22-36
 * (`attention`), layers.py:126-135 (QKNorm), and upstream STDiT3 Attention / MultiHeadCrossAttention
 * (SURVEY.md §8a-S, Appendix A). */
int osb_attn_short(const osb_attn_short_args* args, void* stream);

/* osb_attn_short with an additive fp32 bias by relative position: the score of query token i and key token j is
 * q.k * softmax_scale + bias[h * bias_head_stride + j - i + Lq - 1] (bias: [heads][Lq + Lk - 1], or one shared vector
 * with bias_head_stride = 0), added before the running maximum.  -inf entries mask keys; key blocks that are -inf for
 * every query of a 128-row query tile are skipped, and a row never evaluates -inf - (-inf).  head_dim 64 only; kv_lens
 * and packed short sequences as in osb_attn_short; QK-norm and RoPE arguments keep their meaning.
 * Replaces the self-attention of HF T5Attention (relative_attention_bias, unscaled scores: softmax_scale = 1) and
 * CLIPAttention (causal mask: bias 0 for j <= i, -inf for j > i) run by the reference's text_embedder
 * (opensora/models/text/conditioner.py:10-53). */
int osb_attn_short_bias(const osb_attn_short_args* args, const float* bias, int64_t bias_head_stride, void* stream);

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
 * with the next key tile in flight (open-sora_b200/csrc/attn_sm90.cu).  Replaces mmdit/math.py:22-36. */
int osb_attn_tiles(const osb_attn_tiles_args* args, void* stream);

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
