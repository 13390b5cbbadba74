// Attention on sm_90a: softmax(q k^T * scale) v per (sequence, head), non-causal, exact online softmax.
//
// All entry points run the same flash-attention core.  One CTA (8 warps) owns 128 query rows of one head; every
// warp owns 16 rows and keeps its Q fragments, the running row maximum / sum and the fp32 O accumulator in
// registers.  Key / value tiles sit in shared memory in the head-tile layout (tiles.cuh: 64-column chunks with the
// 128-byte swizzle plus the head-dim tail), so the 16-byte rows that ldmatrix gathers are bank-conflict free for
// K (S = Q K^T) and for V read transposed (O = P V); the tensor core work is mma.sync m16n8k16 (bf16 in, fp32
// accumulate).  P is rounded to bf16 straight from the S accumulator registers, which already have the layout of
// the A operand of the PV product, so S and P never touch shared memory.
//
//   osb_attn_tiles: q / k / v arrive as operand-tile images written by the projection GEMM's head-tile epilogue
//                   (bias, RMSNorm and RoPE applied there); every load is ONE cp.async.bulk of a whole tile completing
//                   on an mbarrier, with the next key tile in flight while the current one is consumed.
//   osb_attn_short: q / k / v are token-layout rows (any strides); the CTA stages them into the same tile layout,
//                   applying per-head RMSNorm and RoPE in fp32 on the way, so q / k / v are read exactly once.
//   osb_attn_short_bias: the osb_attn_short kernel (template kBias) with an fp32 additive bias indexed by the relative
//                   position, bias[h][j - i + Lq - 1], added to the scaled score before the running max (T5's relative
//                   attention bias; a 0 / -inf vector is CLIP's causal mask).  Key blocks whose bias is -inf for every
//                   query of the tile are skipped.
//
// Replaces: opensora/models/mmdit/math.py:22-36 (attention), layers.py:102-135 (QK RMSNorm) and the
// upstream-v1.2 STDiT3 Attention / MultiHeadCrossAttention restated in SURVEY.md App. A.
#include <stdlib.h>

#include "common.cuh"
#include "tiles.cuh"

namespace osb {

constexpr int kAttnThreads = 256;   // 8 warps x 16 query rows
constexpr int kKeyBlock = 64;       // keys per online-softmax step

// ---------------------------------------------------------------------------------------------------------------
// flash core
// ---------------------------------------------------------------------------------------------------------------
template <int D>
struct FlashState {
  static constexpr int DP = HeadTileCfg<D>::DP;
  uint32_t q[DP / 16][4];   // A fragments of this warp's 16 query rows
  float o[DP / 8][4];       // O accumulator: o[j][e] = (row lane/4 + 8 (e/2), column 8 j + 2 (lane%4) + e%2)
  float m[2], l[2];         // running maximum (raw score units) and partial row sum of rows lane/4, lane/4 + 8
};

// Q fragments of rows [16 warp, 16 warp + 16) from a tile image in shared memory (64-column chunks chunk_bytes apart)
template <int D>
__device__ __forceinline__ void flash_load_q(FlashState<D>& f, uint32_t sq, uint32_t chunk_bytes) {
  using Cfg = HeadTileCfg<D>;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row = warp * 16 + (lane & 15);
#pragma unroll
  for (int kk = 0; kk < Cfg::DP / 16; ++kk)
    ldsm_x4(sq + tile_unit_off<Cfg::MAIN>(row, 2 * kk + (lane >> 4), chunk_bytes), f.q[kk][0], f.q[kk][1], f.q[kk][2], f.q[kk][3]);
#pragma unroll
  for (int j = 0; j < Cfg::DP / 8; ++j) f.o[j][0] = f.o[j][1] = f.o[j][2] = f.o[j][3] = 0.f;
  f.m[0] = f.m[1] = -INFINITY;
  f.l[0] = f.l[1] = 0.f;
}

// One block of up to 64 keys: rows [krow0, krow0 + 16 n16) of the K / V tile images (chunk_bytes apart), whose key
// slots are key0 + 0, 1, ...  Row i of this thread (i = 0: lane/4, 1: lane/4 + 8) may only see key slots in
// [lo[i], hi[i]).  sc = softmax scale * log2(e).
// kBias: the score of key slot `key` in row i is s * bscale + bias[key + boff_i] (fp32) and sc = log2(e).
template <int D, bool kBias = false>
__device__ __forceinline__ void flash_block(FlashState<D>& f, uint32_t sk, uint32_t sv, uint32_t chunk_bytes, int krow0,
                                            int n16, int key0, const int (&lo)[2], const int (&hi)[2], float sc,
                                            const float* bias = nullptr, int boff0 = 0, int boff1 = 0, float bscale = 0.f) {
  using Cfg = HeadTileCfg<D>;
  constexpr int NB = kKeyBlock / 8;
  const int lane = threadIdx.x & 31;
  // ---- S = Q K^T ----
  float s[NB][4];
#pragma unroll
  for (int g = 0; g < kKeyBlock / 16; ++g) {
    s[2 * g][0] = s[2 * g][1] = s[2 * g][2] = s[2 * g][3] = 0.f;
    s[2 * g + 1][0] = s[2 * g + 1][1] = s[2 * g + 1][2] = s[2 * g + 1][3] = 0.f;
    if (g >= n16) continue;   // warp-uniform
    const int krow = krow0 + g * 16 + (lane & 7) + ((lane >> 4) << 3);
#pragma unroll
    for (int kk = 0; kk < Cfg::DP / 16; ++kk) {
      uint32_t b0, b1, b2, b3;
      ldsm_x4(sk + tile_unit_off<Cfg::MAIN>(krow, 2 * kk + ((lane >> 3) & 1), chunk_bytes), b0, b1, b2, b3);
      mma_bf16_16816(s[2 * g], f.q[kk], b0, b1);
      mma_bf16_16816(s[2 * g + 1], f.q[kk], b2, b3);
    }
  }
  // ---- mask, block maximum ----
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < NB; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int i = e >> 1;
      const int key = key0 + 8 * j + 2 * (lane & 3) + (e & 1);
      if (j >= 2 * n16 || key < lo[i] || key >= hi[i]) s[j][e] = -INFINITY;
      else if constexpr (kBias) s[j][e] = fmaf(s[j][e], bscale, __ldg(bias + key + (i ? boff1 : boff0)));
      mx[i] = fmaxf(mx[i], s[j][e]);
    }
  }
  float alpha[2], ms[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
    const float mn = fmaxf(f.m[i], mx[i]);
    alpha[i] = (mn == -INFINITY) ? 1.f : fast_exp2((f.m[i] - mn) * sc);   // f.m == -inf: exp2(-inf) = 0
    ms[i] = (mn == -INFINITY) ? 0.f : mn * sc;
    f.m[i] = mn;
    f.l[i] *= alpha[i];
  }
#pragma unroll
  for (int j = 0; j < Cfg::DP / 8; ++j) {
    f.o[j][0] *= alpha[0]; f.o[j][1] *= alpha[0];
    f.o[j][2] *= alpha[1]; f.o[j][3] *= alpha[1];
  }
  // ---- P = exp2(S * sc - max): masked scores are -inf and give 0 ----
#pragma unroll
  for (int j = 0; j < NB; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      s[j][e] = fast_exp2(fmaf(s[j][e], sc, -ms[e >> 1]));
      f.l[e >> 1] += s[j][e];
    }
  }
  // ---- O += P V: the S accumulator of key groups (2g, 2g+1) is the A fragment of k-step g ----
#pragma unroll
  for (int g = 0; g < kKeyBlock / 16; ++g) {
    if (g >= n16) continue;
    const uint32_t a[4] = {pack_bf16x2(s[2 * g][0], s[2 * g][1]), pack_bf16x2(s[2 * g][2], s[2 * g][3]),
                           pack_bf16x2(s[2 * g + 1][0], s[2 * g + 1][1]), pack_bf16x2(s[2 * g + 1][2], s[2 * g + 1][3])};
    const int vrow = krow0 + g * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
#pragma unroll
    for (int dg = 0; dg < Cfg::DP / 16; ++dg) {
      uint32_t b0, b1, b2, b3;
      ldsm_x4_t(sv + tile_unit_off<Cfg::MAIN>(vrow, 2 * dg + (lane >> 4), chunk_bytes), b0, b1, b2, b3);
      mma_bf16_16816(f.o[2 * dg], a, b0, b1);
      mma_bf16_16816(f.o[2 * dg + 1], a, b2, b3);
    }
  }
}

// normalise, round once to bf16 and store row i (0: lane/4, 1: lane/4 + 8) at `dst` (nullptr: row not stored)
template <int D>
__device__ __forceinline__ void flash_store(FlashState<D>& f, __nv_bfloat16* dst0, __nv_bfloat16* dst1) {
  const int lane = threadIdx.x & 31;
  float inv[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = f.l[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv[i] = l > 0.f ? 1.0f / l : 0.f;   // no valid key: zeros, never 0 * garbage
  }
#pragma unroll
  for (int j = 0; j < D / 8; ++j) {
    const int c = 8 * j + 2 * (lane & 3);
    if (dst0) *reinterpret_cast<uint32_t*>(dst0 + c) = pack_bf16x2(f.o[j][0] * inv[0], f.o[j][1] * inv[0]);
    if (dst1) *reinterpret_cast<uint32_t*>(dst1 + c) = pack_bf16x2(f.o[j][2] * inv[1], f.o[j][3] * inv[1]);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// osb_attn_tiles
// ---------------------------------------------------------------------------------------------------------------
struct TileAttnParams {
  const uint8_t* q; const uint8_t* k; const uint8_t* v;   // first tile of head 0
  int64_t q_head_stride, kv_head_stride;                  // bytes
  TileMap qmap;                                           // q tiles <-> rows of `out`
  int32_t q_tile_bytes, q_slot_bytes;                     // TRq * ROW_BYTES; slot: 128 rows
  int32_t kv_tile_bytes, kv_slot_bytes;
  int32_t BK, nkb, Lk;                                    // key-tile rows, key tiles per set, keys per sequence
  int64_t num_seqs, num_sets;
  const int32_t* kv_lens;
  __nv_bfloat16* out;
  int64_t out_ld;
  float scale_log2;
  RowScatter out_sc;        // sequence parallel: output rows go straight to the consuming rank's buffer
};

template <int D>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_tiles_kernel(const TileAttnParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t s0 = smem_u32(smem);
  const uint32_t sQ = s0;
  auto sK = [&](int st) { return s0 + (uint32_t)(p.q_slot_bytes + st * 2 * p.kv_slot_bytes); };
  auto sV = [&](int st) { return sK(st) + (uint32_t)p.kv_slot_bytes; };
  const uint32_t bar = s0 + (uint32_t)(p.q_slot_bytes + 4 * p.kv_slot_bytes);
  const uint32_t q_full = bar;
  auto kv_full = [&](int st) { return bar + 8u + 8u * st; };

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t qtile = blockIdx.x;
  const int head = blockIdx.y;
  const int64_t set = qtile / p.qmap.tps;
  const int qt = (int)(qtile - set * p.qmap.tps);

  // valid key slots of the set (packed tiles: G * Lk, one key range per packed sequence)
  int keys = p.qmap.G > 1 ? p.qmap.G * p.Lk : p.Lk;
  if (p.qmap.G == 1 && p.kv_lens) { const int l = __ldg(p.kv_lens + set); keys = l < keys ? (l < 0 ? 0 : l) : keys; }
  const int nkt = (keys + p.BK - 1) / p.BK;   // key tiles holding valid keys

  if (tid == 0) {
    mbar_init(q_full, 1);
    mbar_init(kv_full(0), 1);
    mbar_init(kv_full(1), 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // the tiles were written by the previous kernel
  const uint8_t* kbase = p.k + (int64_t)head * p.kv_head_stride + set * p.nkb * (int64_t)p.kv_tile_bytes;
  const uint8_t* vbase = p.v + (int64_t)head * p.kv_head_stride + set * p.nkb * (int64_t)p.kv_tile_bytes;
  if (tid == 0) {
    mbar_expect_tx(q_full, (uint32_t)p.q_tile_bytes);
    bulk_load_1d(sQ, p.q + (int64_t)head * p.q_head_stride + qtile * p.q_tile_bytes, (uint32_t)p.q_tile_bytes, q_full);
    for (int st = 0; st < 2 && st < nkt; ++st) {
      mbar_expect_tx(kv_full(st), 2u * (uint32_t)p.kv_tile_bytes);
      bulk_load_1d(sK(st), kbase + (int64_t)st * p.kv_tile_bytes, (uint32_t)p.kv_tile_bytes, kv_full(st));
      bulk_load_1d(sV(st), vbase + (int64_t)st * p.kv_tile_bytes, (uint32_t)p.kv_tile_bytes, kv_full(st));
    }
  }

  // my two query rows: sequence, position, valid key range [lo, hi) in the set's key slots
  int64_t seq[2];
  int pos[2], lo[2], hi[2];
  bool valid[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = warp * 16 + (lane >> 2) + 8 * i;
    lo[i] = hi[i] = 0;
    if (p.qmap.G > 1) {
      const int g = r / p.qmap.L;
      pos[i] = r - g * p.qmap.L;
      seq[i] = set * p.qmap.G + g;
      valid[i] = g < p.qmap.G && seq[i] < p.num_seqs;
      if (valid[i]) { lo[i] = g * p.Lk; hi[i] = lo[i] + p.Lk; }
    } else {
      pos[i] = qt * p.qmap.TR + r;
      seq[i] = set;
      valid[i] = r < p.qmap.TR && pos[i] < p.qmap.L;
      if (valid[i]) hi[i] = keys;
    }
  }

  FlashState<D> f;
  mbar_wait(q_full, 0);
  // rows >= TR of the slot are not part of the tile: they only feed S rows that are never stored
  flash_load_q<D>(f, sQ, (uint32_t)p.qmap.TR * 128u);
  const float sc = p.scale_log2;
  for (int kb = 0; kb < nkt; ++kb) {
    const int st = kb & 1;
    mbar_wait(kv_full(st), (uint32_t)(kb >> 1) & 1u);
    for (int k0 = 0; k0 < p.BK; k0 += kKeyBlock) {
      int n = keys - (kb * p.BK + k0);
      const int cap = p.BK - k0 < kKeyBlock ? p.BK - k0 : kKeyBlock;
      n = n > cap ? cap : n;
      if (n <= 0) break;
      const int lo_b[2] = {lo[0], lo[1]}, hi_b[2] = {hi[0], hi[1]};
      flash_block<D>(f, sK(st), sV(st), (uint32_t)p.BK * 128u, k0, (n + 15) >> 4, kb * p.BK + k0, lo_b, hi_b, sc);
    }
    __syncthreads();   // every warp is done with this stage
    if (tid == 0 && kb + 2 < nkt) {
      mbar_expect_tx(kv_full(st), 2u * (uint32_t)p.kv_tile_bytes);
      bulk_load_1d(sK(st), kbase + (int64_t)(kb + 2) * p.kv_tile_bytes, (uint32_t)p.kv_tile_bytes, kv_full(st));
      bulk_load_1d(sV(st), vbase + (int64_t)(kb + 2) * p.kv_tile_bytes, (uint32_t)p.kv_tile_bytes, kv_full(st));
    }
  }
  pdl_launch_dependents();

  __nv_bfloat16* dst[2] = {nullptr, nullptr};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (!valid[i]) continue;
    int64_t orow = row_of_token(p.qmap, seq[i], pos[i]);
    __nv_bfloat16* obase = p.out;
    if (p.out_sc.mode != 0) {
      int peer;
      scatter_row(p.out_sc, orow, peer, orow);
      obase = static_cast<__nv_bfloat16*>(scatter_base(p.out_sc, peer));
    }
    dst[i] = obase + orow * p.out_ld + (int64_t)head * D;
  }
  flash_store<D>(f, dst[0], dst[1]);
}

template <int D>
static int attn_tiles_launch(TileAttnParams& p, int H, cudaStream_t stream) {
  using Cfg = HeadTileCfg<D>;
  p.q_tile_bytes = p.qmap.TR * Cfg::ROW_BYTES;
  p.q_slot_bytes = 128 * Cfg::ROW_BYTES;   // the Q fragments are read for 128 rows whatever TR is
  p.kv_tile_bytes = p.BK * Cfg::ROW_BYTES;
  p.kv_slot_bytes = (p.kv_tile_bytes + 127) / 128 * 128;
  const int smem = p.q_slot_bytes + 4 * p.kv_slot_bytes + 64;
  const int64_t qtiles = p.num_sets * p.qmap.tps;
  if (qtiles >= (1ll << 31) || H > 65535) { set_error("osb_attn_tiles: problem too large (%lld query tiles)", (long long)qtiles); return OSB_ERR_UNSUPPORTED; }
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)qtiles, (unsigned)H), dim3(kAttnThreads), smem, stream, attr);
  OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_tiles_kernel<D>, p));
  count_launch();
  return OSB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// osb_attn_short
// ---------------------------------------------------------------------------------------------------------------
struct AttnParams {
  const __nv_bfloat16* q; const __nv_bfloat16* k; const __nv_bfloat16* v; __nv_bfloat16* out;
  int64_t q_ld, k_ld, v_ld, out_ld;
  int64_t num_seqs, seqs_per_batch;
  int64_t q_bs, q_ss, q_ts, k_bs, k_ss, k_ts;
  int32_t Lq, Lk;
  const int32_t* kv_lens;
  const __nv_bfloat16* qw; const __nv_bfloat16* kw;
  const __nv_bfloat16* qw2; const __nv_bfloat16* kw2;  // weights for tokens >= norm_split (joint txt|img sequences)
  int32_t norm_split;
  float eps;
  const float* cos; const float* sin;
  int32_t rope_half;     // 1: rotate-half pairing (i, i + D/2) (HF / Liger layout), 0: interleaved pairs (2i, 2i+1)
  float scale_log2;      // softmax_scale * log2(e)
  int32_t G;             // sequences packed per 128-row query tile (1 when Lq >= 128)
  int32_t tiles_per_seq; // query tiles per sequence (G == 1)
  const float* bias;     // kBias: fp32 [heads][Lq + Lk - 1], head h at bias + h * bias_hs
  int64_t bias_hs;
  float scale;           // kBias: softmax_scale (the bias is added to the scaled score)
};

__device__ __forceinline__ void unpack8(const uint4& t, float* x) {
  const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = unpack_bf16x2(tw[e]);
    x[2 * e] = f.x;
    x[2 * e + 1] = f.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* x) {
  uint4 o;
  o.x = pack_bf16x2(x[0], x[1]);
  o.y = pack_bf16x2(x[2], x[3]);
  o.z = pack_bf16x2(x[4], x[5]);
  o.w = pack_bf16x2(x[6], x[7]);
  return o;
}

// One head row (U raw bf16x8 units) -> optional RMSNorm scale r*w and RoPE in fp32 -> bf16 -> row `row` of a tile
// image in shared memory (64-column chunks chunk_bytes apart, head-dim tail zero padded).  Works unit by unit (a
// rotate-half pair of units at a time) so that no fp32 copy of the whole row is live.
template <int D>
__device__ __forceinline__ void stage_row(uint4 (&raw)[HeadTileCfg<D>::U], bool norm, float eps, const __nv_bfloat16* w,
                                          const float* cosr, const float* sinr, bool rope_half, uint8_t* tile,
                                          uint32_t chunk_bytes, int row) {
  using Cfg = HeadTileCfg<D>;
  constexpr int U = Cfg::U;
  float r = 1.f;
  if (norm) {
    float ss = 0.f;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float x[8];
      unpack8(raw[u], x);
#pragma unroll
      for (int e = 0; e < 8; ++e) ss += x[e] * x[e];
    }
    r = rsqrtf(ss * (1.0f / D) + eps);
  }
  auto scale = [&](int u, float* x) {
    unpack8(raw[u], x);
    if (norm) {
      float wf[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(w) + u), wf);
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] *= r * wf[e];
    }
  };
  if (cosr != nullptr && rope_half) {   // LigerRopeFunction (math.py:27): element i pairs with i + D/2
#pragma unroll
    for (int u = 0; u < U / 2; ++u) {
      float x1[8], x2[8];
      scale(u, x1);
      scale(u + U / 2, x2);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float c = __ldg(cosr + 8 * u + e), sn = __ldg(sinr + 8 * u + e);
        const float a = x1[e], b = x2[e];
        x1[e] = a * c - b * sn;
        x2[e] = b * c + a * sn;
      }
      raw[u] = pack8(x1);
      raw[u + U / 2] = pack8(x2);
    }
  } else if (norm || cosr != nullptr) {
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float x[8];
      scale(u, x);
      if (cosr != nullptr) {   // interleaved pairs (2i, 2i+1) (math.py:60-65)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float c = __ldg(cosr + 4 * u + i), sn = __ldg(sinr + 4 * u + i);
          const float a = x[2 * i], b = x[2 * i + 1];
          x[2 * i] = a * c - b * sn;
          x[2 * i + 1] = b * c + a * sn;
        }
      }
      raw[u] = pack8(x);
    }
  }
#pragma unroll
  for (int u = 0; u < Cfg::UP; ++u)
    *reinterpret_cast<uint4*>(tile + tile_unit_off<Cfg::MAIN>(row, u, chunk_bytes)) = u < U ? raw[u] : make_uint4(0, 0, 0, 0);
}

template <int D, bool kBias>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_short_kernel(const AttnParams p) {
  using Cfg = HeadTileCfg<D>;
  constexpr int U = Cfg::U;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;                                    // [128 x DP] tile image
  uint8_t* sK = smem + 128 * Cfg::ROW_BYTES;             // [64 x DP]
  uint8_t* sV = sK + kKeyBlock * Cfg::ROW_BYTES;         // [64 x DP]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t unit = blockIdx.x;
  const int h = blockIdx.y;

  int64_t seq0;
  int qt = 0;
  if (p.G > 1) seq0 = unit * p.G;
  else { seq0 = unit / p.tiles_per_seq; qt = (int)(unit - seq0 * p.tiles_per_seq); }
  auto row_of = [&](int64_t seq, int tok, int64_t bs, int64_t ss, int64_t ts) {
    const int64_t b = seq / p.seqs_per_batch, j = seq - b * p.seqs_per_batch;
    return b * bs + j * ss + (int64_t)tok * ts;
  };

  __shared__ int s_nkeys;
  if (tid == 0) s_nkeys = 0;
  __syncthreads();
  pdl_wait();   // q, k, v were written by the previous kernel
  // ---- stage Q (128 rows) ----
  for (int r = tid; r < 128; r += kAttnThreads) {
    const int g = p.G > 1 ? r / p.Lq : 0;
    const int tok = p.G > 1 ? r - g * p.Lq : qt * 128 + r;
    const int64_t seq = seq0 + g;
    uint4 raw[U];
    const bool ok = g < p.G && seq < p.num_seqs && tok < p.Lq;
    if (ok) {
      const uint4* src = reinterpret_cast<const uint4*>(p.q + row_of(seq, tok, p.q_bs, p.q_ss, p.q_ts) * p.q_ld + (int64_t)h * D);
#pragma unroll
      for (int u = 0; u < U; ++u) raw[u] = __ldg(src + u);
    } else {
#pragma unroll
      for (int u = 0; u < U; ++u) raw[u] = make_uint4(0, 0, 0, 0);
    }
    const __nv_bfloat16* w = (p.qw2 != nullptr && tok >= p.norm_split) ? p.qw2 : p.qw;
    const bool rope = ok && p.cos != nullptr;
    stage_row<D>(raw, ok && p.qw != nullptr, p.eps, w, rope ? p.cos + (int64_t)tok * (D / 2) : nullptr,
                 rope ? p.sin + (int64_t)tok * (D / 2) : nullptr, p.rope_half, sQ, 128u * 128u, r);
  }

  // my two query rows: valid key slots [lo, hi) and output pointers
  int lo[2], hi[2];
  int boff[2] = {0, 0};   // kBias: bias index of key slot `key` = key + boff (= key token - query token + Lq - 1)
  __nv_bfloat16* dst[2] = {nullptr, nullptr};
  int nkeys = 0;   // key slots any row of the CTA may see
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = warp * 16 + (lane >> 2) + 8 * i;
    const int g = p.G > 1 ? r / p.Lq : 0;
    const int tok = p.G > 1 ? r - g * p.Lq : qt * 128 + r;
    const int64_t seq = seq0 + g;
    lo[i] = hi[i] = 0;
    if (g < p.G && seq < p.num_seqs && tok < p.Lq) {
      int len = p.kv_lens ? p.kv_lens[seq] : p.Lk;
      len = len < p.Lk ? (len < 0 ? 0 : len) : p.Lk;
      lo[i] = g * p.Lk;
      hi[i] = lo[i] + len;
      if constexpr (kBias) boff[i] = p.Lq - 1 - tok - lo[i];
      dst[i] = p.out + row_of(seq, tok, p.q_bs, p.q_ss, p.q_ts) * p.out_ld + (int64_t)h * D;
    }
    nkeys = hi[i] > nkeys ? hi[i] : nkeys;
  }
  atomicMax(&s_nkeys, nkeys);
  __syncthreads();   // (also: the Q tile is staged)
  nkeys = s_nkeys;

  FlashState<D> f;
  flash_load_q<D>(f, smem_u32(sQ), 128u * 128u);
  const float sc = p.scale_log2;
  const float* bh = nullptr;
  if constexpr (kBias) bh = p.bias + (int64_t)h * p.bias_hs;
  for (int k0 = 0; k0 < nkeys; k0 += kKeyBlock) {
    if constexpr (kBias) {
      // Skip the block when the bias is -inf for every (query, key) pair of the tile: the pairs cover the relative
      // positions [k0 - last query, block end - first query], at most 64 + 127 of them, one per thread.
      if (p.G == 1) {
        const int iq0 = qt * 128, iq1 = (iq0 + 128 < p.Lq ? iq0 + 128 : p.Lq) - 1;
        const int kend = k0 + kKeyBlock < nkeys ? k0 + kKeyBlock : nkeys;
        const int d0 = k0 - iq1 + p.Lq - 1, d1 = kend - 1 - iq0 + p.Lq - 1;
        const bool live = d0 + tid <= d1 && __ldg(bh + d0 + tid) != -INFINITY;
        if (!__syncthreads_or(live)) continue;
      }
    }
    // ---- stage keys / values [k0, k0 + 64): K with RMSNorm + RoPE, V as is ----
    for (int s = tid; s < kKeyBlock; s += kAttnThreads) {
      const int slot = k0 + s;
      const int kg = slot / p.Lk, ktok = slot - kg * p.Lk;
      const int64_t kseq = seq0 + kg;
      const bool ok = slot < nkeys && kseq < p.num_seqs;
      int64_t krow = 0;
      if (ok) krow = row_of(kseq, ktok, p.k_bs, p.k_ss, p.k_ts);
      uint4 t[U];
      {
        const uint4* ks = reinterpret_cast<const uint4*>(p.k + krow * p.k_ld + (int64_t)h * D);
#pragma unroll
        for (int u = 0; u < U; ++u) t[u] = ok ? __ldg(ks + u) : make_uint4(0, 0, 0, 0);
        const __nv_bfloat16* w = (p.kw2 != nullptr && ktok >= p.norm_split) ? p.kw2 : p.kw;
        const bool rope = ok && p.cos != nullptr;
        stage_row<D>(t, ok && p.kw != nullptr, p.eps, w, rope ? p.cos + (int64_t)ktok * (D / 2) : nullptr,
                     rope ? p.sin + (int64_t)ktok * (D / 2) : nullptr, p.rope_half, sK, kKeyBlock * 128u, s);
      }
      {
        const uint4* vs = reinterpret_cast<const uint4*>(p.v + krow * p.v_ld + (int64_t)h * D);
#pragma unroll
        for (int u = 0; u < U; ++u) t[u] = ok ? __ldg(vs + u) : make_uint4(0, 0, 0, 0);
        stage_row<D>(t, false, 0.f, nullptr, nullptr, nullptr, false, sV, kKeyBlock * 128u, s);
      }
    }
    __syncthreads();
    const int n = nkeys - k0 < kKeyBlock ? nkeys - k0 : kKeyBlock;
    if constexpr (kBias)
      flash_block<D, true>(f, smem_u32(sK), smem_u32(sV), kKeyBlock * 128u, 0, (n + 15) >> 4, k0, lo, hi, sc, bh, boff[0],
                           boff[1], p.scale);
    else
      flash_block<D>(f, smem_u32(sK), smem_u32(sV), kKeyBlock * 128u, 0, (n + 15) >> 4, k0, lo, hi, sc);
    __syncthreads();   // the next block overwrites sK / sV
  }
  pdl_launch_dependents();
  flash_store<D>(f, dst[0], dst[1]);
}

template <int D, bool kBias = false>
static int attn_short_launch(const AttnParams& p, int64_t units, int H, cudaStream_t stream) {
  using Cfg = HeadTileCfg<D>;
  const int smem = (128 + 2 * kKeyBlock) * Cfg::ROW_BYTES;
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)units, (unsigned)H), dim3(kAttnThreads), smem, stream, attr);
  OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_short_kernel<D, kBias>, p));
  count_launch();
  return OSB_OK;
}

int attn_init() {
  constexpr int kMax = 200 * 1024;   // largest carve-up: 128-row Q slot + two K/V stages of 128-row D = 128 tiles
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_short_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_short_kernel<72, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_short_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_short_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_kernel<72>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  return OSB_OK;
}

}  // namespace osb

extern "C" int64_t osb_head_tiles_per_head(const osb_tile_map* m, int64_t rows) {
  if (m == nullptr || m->L <= 0 || m->tile_rows <= 0) return -1;
  const int64_t seqs = rows / m->L;
  if (m->G > 1) return (seqs + m->G - 1) / m->G;
  return seqs * m->tps;
}

extern "C" int osb_attn_tiles(const osb_attn_tiles_args* a, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(a != nullptr, "osb_attn_tiles: null args");
  OSB_REQUIRE(a->q_tiles && a->k_tiles && a->v_tiles && (a->out || a->out_scatter), "osb_attn_tiles: null tensor");
  const int D = a->head_dim;
  OSB_REQUIRE(D == 64 || D == 72 || D == 128, "osb_attn_tiles: head_dim %d not built (64, 72, 128)", D);
  const osb_tile_map& m = a->q_map;
  OSB_REQUIRE(m.mode == 0 || m.mode == 1, "osb_attn_tiles: unknown tile map mode %d", m.mode);
  OSB_REQUIRE(m.L > 0 && m.G >= 1 && m.tile_rows > 0 && m.tile_rows <= 128 && m.tile_rows % 8 == 0,
              "osb_attn_tiles: bad q tile map (L %d G %d rows %d)", m.L, m.G, m.tile_rows);
  OSB_REQUIRE(m.G == 1 ? (m.tps == (m.L + m.tile_rows - 1) / m.tile_rows) : (m.G * m.L <= m.tile_rows && m.tps == 1),
              "osb_attn_tiles: q tile map inconsistent (L %d G %d tps %d rows %d)", m.L, m.G, m.tps, m.tile_rows);
  OSB_REQUIRE(m.mode == 0 || (m.S > 0 && m.T == m.L), "osb_attn_tiles: temporal map needs S > 0 and T == L");
  OSB_REQUIRE(a->kv_tile_rows >= 16 && a->kv_tile_rows <= 128 && a->kv_tile_rows % 16 == 0,
              "osb_attn_tiles: key tiles must have 16..128 rows in multiples of 16, got %d", a->kv_tile_rows);
  OSB_REQUIRE(a->Lk > 0 && a->kv_tiles_per_set >= 1 && (int64_t)a->kv_tiles_per_set * a->kv_tile_rows >= (int64_t)(m.G > 1 ? m.G : 1) * a->Lk,
              "osb_attn_tiles: %d key tiles of %d rows cannot hold %d keys", a->kv_tiles_per_set, a->kv_tile_rows, a->Lk);
  OSB_REQUIRE(m.G == 1 || (a->kv_tiles_per_set == 1), "osb_attn_tiles: packed sequences use one key tile per set");
  OSB_REQUIRE(a->num_seqs > 0 && a->num_heads > 0, "osb_attn_tiles: empty problem");
  OSB_REQUIRE(a->out_ld % 8 == 0 && (reinterpret_cast<uintptr_t>(a->out) & 15) == 0, "osb_attn_tiles: out must be 16-byte aligned");
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(a->q_tiles) | reinterpret_cast<uintptr_t>(a->k_tiles) | reinterpret_cast<uintptr_t>(a->v_tiles)) & 15) == 0 &&
              a->q_head_stride % 16 == 0 && a->kv_head_stride % 16 == 0, "osb_attn_tiles: tile buffers must be 16-byte aligned");

  TileAttnParams p = {};
  p.q = static_cast<const uint8_t*>(a->q_tiles);
  p.k = static_cast<const uint8_t*>(a->k_tiles);
  p.v = static_cast<const uint8_t*>(a->v_tiles);
  p.q_head_stride = a->q_head_stride; p.kv_head_stride = a->kv_head_stride;
  p.qmap.mode = m.mode; p.qmap.L = m.L; p.qmap.S = m.S; p.qmap.T = m.T; p.qmap.G = m.G; p.qmap.tps = m.tps; p.qmap.TR = m.tile_rows;
  p.BK = a->kv_tile_rows; p.nkb = a->kv_tiles_per_set; p.Lk = a->Lk;
  p.num_seqs = a->num_seqs;
  p.num_sets = m.G > 1 ? (a->num_seqs + m.G - 1) / m.G : a->num_seqs;
  p.kv_lens = a->kv_lens;
  p.out = static_cast<__nv_bfloat16*>(a->out);
  p.out_ld = a->out_ld;
  p.scale_log2 = a->softmax_scale * 1.4426950408889634f;
  {
    const int64_t out_rows = a->num_seqs * m.L;
    const int rc = make_row_scatter(&p.out_sc, a->out_scatter, out_rows, "osb_attn_tiles");
    if (rc) return rc;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (D == 64) return attn_tiles_launch<64>(p, a->num_heads, s);
  if (D == 72) return attn_tiles_launch<72>(p, a->num_heads, s);
  return attn_tiles_launch<128>(p, a->num_heads, s);
}

// Argument checks and launch shared by osb_attn_short and osb_attn_short_bias (bias == nullptr: the plain kernel).
static int attn_short_entry(const osb_attn_short_args* a, const float* bias, int64_t bias_head_stride, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(a != nullptr, "osb_attn_short: null args");
  OSB_REQUIRE(a->q && a->k && a->v && a->out, "osb_attn_short: null tensor");
  OSB_REQUIRE(a->Lq > 0 && a->Lk > 0 && a->num_seqs > 0 && a->num_heads > 0,
              "osb_attn_short: empty problem");
  OSB_REQUIRE(a->seqs_per_batch > 0, "osb_attn_short: seqs_per_batch must be positive");
  const int D = a->head_dim;
  OSB_REQUIRE(D == 64 || D == 72 || D == 128, "osb_attn_short: head_dim %d not built (64, 72, 128)", D);
  OSB_REQUIRE((a->q_ld % 8) == 0 && (a->k_ld % 8) == 0 && (a->v_ld % 8) == 0 && (a->out_ld % 8) == 0,
              "osb_attn_short: leading dimensions must be multiples of 8 elements");
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(a->q) | reinterpret_cast<uintptr_t>(a->k) |
                reinterpret_cast<uintptr_t>(a->v) | reinterpret_cast<uintptr_t>(a->out)) & 15) == 0,
              "osb_attn_short: tensors must be 16-byte aligned");
  OSB_REQUIRE((a->q_norm_w == nullptr) == (a->k_norm_w == nullptr), "osb_attn_short: q/k norm weights must come together");
  OSB_REQUIRE((a->rope_cos == nullptr) == (a->rope_sin == nullptr), "osb_attn_short: rope cos/sin must come together");
  OSB_REQUIRE((a->q_norm_w2 == nullptr) == (a->k_norm_w2 == nullptr) && (a->q_norm_w2 == nullptr || a->q_norm_w != nullptr),
              "osb_attn_short: the second norm weight pair needs the first");
  OSB_REQUIRE(a->rope_cos == nullptr || ((reinterpret_cast<uintptr_t>(a->rope_cos) | reinterpret_cast<uintptr_t>(a->rope_sin)) & 15) == 0,
              "osb_attn_short: rope tables must be 16-byte aligned");

  AttnParams p;
  p.q = static_cast<const __nv_bfloat16*>(a->q);
  p.k = static_cast<const __nv_bfloat16*>(a->k);
  p.v = static_cast<const __nv_bfloat16*>(a->v);
  p.out = static_cast<__nv_bfloat16*>(a->out);
  p.q_ld = a->q_ld; p.k_ld = a->k_ld; p.v_ld = a->v_ld; p.out_ld = a->out_ld;
  p.num_seqs = a->num_seqs; p.seqs_per_batch = a->seqs_per_batch;
  p.q_bs = a->q_batch_stride; p.q_ss = a->q_seq_stride; p.q_ts = a->q_tok_stride;
  p.k_bs = a->k_batch_stride; p.k_ss = a->k_seq_stride; p.k_ts = a->k_tok_stride;
  p.Lq = a->Lq; p.Lk = a->Lk; p.kv_lens = a->kv_lens;
  p.qw = static_cast<const __nv_bfloat16*>(a->q_norm_w);
  p.kw = static_cast<const __nv_bfloat16*>(a->k_norm_w);
  p.qw2 = static_cast<const __nv_bfloat16*>(a->q_norm_w2);
  p.kw2 = static_cast<const __nv_bfloat16*>(a->k_norm_w2);
  p.norm_split = a->norm_split;
  p.eps = a->norm_eps;
  p.cos = a->rope_cos; p.sin = a->rope_sin;
  p.rope_half = a->rope_cos != nullptr && a->rope_half ? 1 : 0;
  OSB_REQUIRE(!p.rope_half || (D % 16 == 0), "osb_attn_short: rotate-half RoPE needs head_dim %% 16 == 0");
  p.scale_log2 = a->softmax_scale * 1.4426950408889634f;
  int64_t units;
  if (a->Lq >= 128) {
    p.G = 1;
    p.tiles_per_seq = (a->Lq + 127) / 128;
    units = a->num_seqs * p.tiles_per_seq;
  } else {   // short sequences: 128 / Lq of them share a query tile (block-diagonal mask)
    p.G = 128 / a->Lq;
    p.tiles_per_seq = 1;
    units = (a->num_seqs + p.G - 1) / p.G;
  }
  OSB_REQUIRE((int64_t)p.G * a->Lk < (1ll << 31), "osb_attn_short: too many keys per query tile");
  OSB_REQUIRE(units <= 0x7fffffff && a->num_heads <= 65535, "osb_attn_short: grid too large");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  p.bias = bias;
  p.bias_hs = bias_head_stride;
  p.scale = a->softmax_scale;
  if (bias != nullptr) {
    OSB_REQUIRE(D == 64, "osb_attn_short_bias: head_dim %d not built (64)", D);
    OSB_REQUIRE(bias_head_stride >= 0, "osb_attn_short_bias: negative bias_head_stride");
    p.scale_log2 = 1.4426950408889634f;   // the scale is applied before the bias is added
    return attn_short_launch<64, true>(p, units, a->num_heads, s);
  }
  if (D == 64) return attn_short_launch<64>(p, units, a->num_heads, s);
  if (D == 72) return attn_short_launch<72>(p, units, a->num_heads, s);
  return attn_short_launch<128>(p, units, a->num_heads, s);
}

extern "C" int osb_attn_short(const osb_attn_short_args* a, void* stream) { return attn_short_entry(a, nullptr, 0, stream); }

extern "C" int osb_attn_short_bias(const osb_attn_short_args* a, const float* bias, int64_t bias_head_stride, void* stream) {
  if (bias == nullptr) { osb::set_error("osb_attn_short_bias: null bias"); return OSB_ERR_INVALID; }
  return attn_short_entry(a, bias, bias_head_stride, stream);
}
