// FP8 (e4m3) attention on sm_90a (include/osb200.h): MMDiT's joint txt|img self-attention (osb_attn_fp8) and the
// head-tile attention of STDiT3 (osb_head_tiles_fp8 / osb_attn_tiles_fp8; tile format in tiles.cuh).
//
// Both attention kernels have one structure: one CTA per (128 queries, head), 3 warpgroups.  Warpgroup 0 (24 registers)
// has one thread that loads the Q tile once and streams K, V^T and their scales through a 4-stage mbarrier ring;
// warpgroups 1 and 2 (240 registers) own 64 query rows each and run fp8_flash_block per key block: S = Q K^T by wgmma
// with both operands in shared memory, the online softmax in registers, P8 = e4m3(256 p) packed straight from the S
// accumulator into the register A fragment of the PV wgmma (the vt8 key permutation makes the two layouts agree), PV
// into a partial accumulator that is promoted into the fp32 O.  They differ in their producers and in the promotion.
//
// osb_attn_fp8, three launches, each with PDL:
//   attn_fp8_prep_kernel   one CTA per (64 tokens, sequence x head).  Each of 128 threads stages one q or k row exactly
//                          as osb_attn_short does (stage.cuh: RMSNorm with the stream's weight, RoPE, one rounding to
//                          bf16), then writes its e4m3 codes and per-row scale.  The same CTA reduces v's per-channel
//                          amax over its 64 tokens and publishes it with atomicMax on the float bits (non-negative floats
//                          order like their bit patterns, so the result does not depend on the order of the atomics).
//   attn_fp8_vpack_kernel  one CTA per (128 keys, sequence x head): v / s_v as e4m3, transposed through shared memory
//                          to [channel][key] with the key permutation of the header inside every 32-key group.
//   attn_fp8_kernel        the producer loads by 2-D TMA (128-byte swizzle rows = 128 e4m3) and bulk-copies the 128 key
//                          scales; O = alpha O + partial, s_v (one scale per channel for the whole sequence) applied at
//                          the output.  This kernel also zeroes the v amax scratch for the next call, after the V pack
//                          read it.
// osb_head_tiles_fp8 / osb_attn_tiles_fp8:
//   head_tiles_fp8_kernel  one CTA of 128 threads per (tile, head, kind).  q / k: thread r quantizes row r of the bf16
//                          tile (per-row scale) and stores its 128-byte swizzled e4m3 row.  v: the tile is staged in
//                          shared memory, thread c reduces channel c over the tile's rows and stores the channel's
//                          codes in the vt8 key order.
//   attn_tiles_fp8_kernel  the producer bulk-copies the tile images with their scales; ceil(D / 32) k32 steps of QK^T,
//                          PV with N = D, O = alpha O + s_v (.) partial (v scales per key tile).  The output rows are
//                          addressed as attn_tiles_kernel addresses them (tiles.cuh: inverse q map, optional scatter).
#include "common.cuh"
#include "stage.cuh"
#include "tiles.cuh"
#include "wgmma.cuh"

namespace osb {

constexpr int kF8D = 128;          // head_dim
constexpr int kF8KB = 128;         // keys per block, and the granularity of Lpad
constexpr int kF8Stages = 4;
constexpr int kF8Threads = 384;    // producer warpgroup + two consumer warpgroups
constexpr int kF8TileBytes = 128 * 128;
constexpr int kF8Smem = 1024 + kF8TileBytes + kF8Stages * (2 * kF8TileBytes + 512) + 8 * (1 + 2 * kF8Stages);

constexpr int kTF8Stages = 4;
constexpr int kTF8StageBytes = 2 * kTileF8Bytes + 1024;   // K tile, V tile (D <= 128 rows), k scales, v scales
constexpr int kTF8Smem = 1024 + kTileF8Bytes + kTF8Stages * kTF8StageBytes + 8 * (1 + 2 * kTF8Stages);

// ---------------------------------------------------------------------------------------------------------------
// e4m3 packing and the flash step shared by both paths
// ---------------------------------------------------------------------------------------------------------------
// 16 values -> their e4m3 codes at scale s (x / s), in order: one 16-byte unit of a q / k row
__device__ __forceinline__ uint4 e4m3x16(const float (&x)[16], float s) {
  uint4 o;
  o.x = e4m3x2(x[0] / s, x[1] / s) | (e4m3x2(x[2] / s, x[3] / s) << 16);
  o.y = e4m3x2(x[4] / s, x[5] / s) | (e4m3x2(x[6] / s, x[7] / s) << 16);
  o.z = e4m3x2(x[8] / s, x[9] / s) | (e4m3x2(x[10] / s, x[11] / s) << 16);
  o.w = e4m3x2(x[12] / s, x[13] / s) | (e4m3x2(x[14] / s, x[15] / s) << 16);
  return o;
}

// the codes of channel c at vt8 positions [pos0, pos0 + 16) at scale s: key vt8_key(pos) of a [key][channel] bf16 tile
// in shared memory.  One 16-byte unit of a v^T row.
template <int C>
__device__ __forceinline__ uint4 vt8_pack16(const __nv_bfloat16 (*tile)[C], int c, int pos0, float s) {
  uint32_t w[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int pos = pos0 + 4 * r;
    const float x0 = __bfloat162float(tile[vt8_key(pos)][c]), x1 = __bfloat162float(tile[vt8_key(pos + 1)][c]);
    const float x2 = __bfloat162float(tile[vt8_key(pos + 2)][c]), x3 = __bfloat162float(tile[vt8_key(pos + 3)][c]);
    w[r] = e4m3x2(x0 / s, x1 / s) | (e4m3x2(x2 / s, x3 / s) << 16);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// One key block of a consumer warpgroup (64 query rows; this thread: rows r_loc and r_loc + 8, accumulator fragment
// x[4 j + 2 hh + e] = (row r_loc + 8 hh, column 8 j + 2 (lane % 4) + e)).  The K tile (128 rows of 128 e4m3) and the
// V^T tile (D rows in the vt8 key order) are at k_smem / v_smem, the stage's 128 key scales at k_scale, its D value
// scales at v_scale (kScaleV only); sq = s_q * softmax_scale * log2(e) per row.  Key slot slot0 + col is seen by row hh
// iff col < BK and lo[hh] <= slot < hi[hh].  The stage is released once the PV product retired.  Promotion of the
// partial: o += part (the value scales are applied at the output) or, kScaleV, o += s_v (.) part.
template <int D, bool kScaleV>
__device__ __forceinline__ void fp8_flash_block(float (&o)[D / 2], float (&part)[D / 2], float (&s)[64], float (&m)[2],
                                                float (&l)[2], uint64_t dq, uint32_t k_smem, uint32_t v_smem,
                                                const float* k_scale, const float* v_scale, const float (&sq)[2], int slot0,
                                                int BK, const int (&lo)[2], const int (&hi)[2], uint32_t empty) {
  constexpr int KSTEPS = (D + 31) / 32;   // k32 steps of QK^T: the codes past D are zero
  const int quad = threadIdx.x & 3;
  // ---- S = Q K^T (+32 bytes = +2 in the descriptors per k32 step) ----
  const uint64_t dk = make_sw128_kmajor_desc(k_smem);
  wgmma_fence_regs(s);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) WgmmaFp8<128>::mma(s, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(s);
  // ---- scores in log2 units, masks, running maximum ----
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float2 sk = *reinterpret_cast<const float2*>(k_scale + 8 * j + 2 * quad);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * j + 2 * quad + e, slot = slot0 + col;
        float v = s[4 * j + 2 * hh + e] * sq[hh] * (e ? sk.y : sk.x);
        if (col >= BK || slot < lo[hh] || slot >= hi[hh]) v = -INFINITY;
        s[4 * j + 2 * hh + e] = v;
        mx[hh] = fmaxf(mx[hh], v);
      }
    }
  }
  float alpha[2], ms[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
    const float mn = fmaxf(m[hh], mx[hh]);
    alpha[hh] = mn == -INFINITY ? 1.f : fast_exp2(m[hh] - mn);   // m == -inf (no key seen yet): 0
    ms[hh] = mn == -INFINITY ? 0.f : mn;                          // a row with no valid key: every p is 0
    m[hh] = mn;
    l[hh] *= alpha[hh];
  }
  // ---- p = exp2(S - m) (masked: 0), l += p, P8 = e4m3(256 p) in the A fragment order ----
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const float pv = fast_exp2(s[i] - ms[(i >> 1) & 1]);
    l[(i >> 1) & 1] += pv;
    s[i] = 256.f * pv;
  }
  uint32_t pa[4][4];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    pa[g][0] = e4m3x2(s[16 * g + 0], s[16 * g + 1]) | (e4m3x2(s[16 * g + 4], s[16 * g + 5]) << 16);
    pa[g][1] = e4m3x2(s[16 * g + 2], s[16 * g + 3]) | (e4m3x2(s[16 * g + 6], s[16 * g + 7]) << 16);
    pa[g][2] = e4m3x2(s[16 * g + 8], s[16 * g + 9]) | (e4m3x2(s[16 * g + 12], s[16 * g + 13]) << 16);
    pa[g][3] = e4m3x2(s[16 * g + 10], s[16 * g + 11]) | (e4m3x2(s[16 * g + 14], s[16 * g + 15]) << 16);
  }
  // ---- partial = P8 V8 (tensor core), then the promotion into O in fp32 ----
  // the v scales are read before the product: once the warpgroup's wgmma retired, every warp is done with the stage
  float2 sv[kScaleV ? D / 8 : 1];
  if constexpr (kScaleV) {
#pragma unroll
    for (int j = 0; j < D / 8; ++j) sv[j] = *reinterpret_cast<const float2*>(v_scale + 8 * j + 2 * quad);
  }
  const uint64_t dv = make_sw128_kmajor_desc(v_smem);
  wgmma_fence_regs(part);
  wgmma_fence();
#pragma unroll
  for (int g = 0; g < 4; ++g) WgmmaFp8RegA<D>::mma(part, pa[g], dv + (uint64_t)(2 * g), g > 0 ? 1u : 0u);
  wgmma_commit();
#pragma unroll
  for (int j = 0; j < D / 8; ++j) {   // overlaps the PV product
    o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0];
    o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
  }
  wgmma_wait<0>();
  wgmma_fence_regs(part);
#pragma unroll
  for (int g = 0; g < 4; ++g) fence_regs_u32(pa[g]);   // the A registers stay untouched until the product retired
  if ((threadIdx.x & 127) == 0) mbar_arrive(empty);
#pragma unroll
  for (int j = 0; j < D / 8; ++j) {
    if constexpr (kScaleV) {
      o[4 * j] += sv[j].x * part[4 * j]; o[4 * j + 1] += sv[j].y * part[4 * j + 1];
      o[4 * j + 2] += sv[j].x * part[4 * j + 2]; o[4 * j + 3] += sv[j].y * part[4 * j + 3];
    } else {
      o[4 * j] += part[4 * j]; o[4 * j + 1] += part[4 * j + 1];
      o[4 * j + 2] += part[4 * j + 2]; o[4 * j + 3] += part[4 * j + 3];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// osb_attn_fp8
// ---------------------------------------------------------------------------------------------------------------
struct Fp8AttnPrep {
  const __nv_bfloat16* q; const __nv_bfloat16* k; const __nv_bfloat16* v;
  int64_t q_ld, k_ld, v_ld;
  int64_t q_bs, q_ts, k_bs, k_ts;   // row of token t of sequence b: b * bs + t * ts (k's map also addresses v)
  int32_t L, Lpad, H;
  const __nv_bfloat16* qw; const __nv_bfloat16* kw;
  const __nv_bfloat16* qw2; const __nv_bfloat16* kw2;
  int32_t norm_split;
  float eps;
  const float* cos; const float* sin;
  int32_t rope_half;
  uint8_t* q8; uint8_t* k8; uint8_t* vt8;
  float* s_q; float* s_k; float* s_v; float* v_amax;
};

struct Fp8AttnMain {
  const float* s_q; const float* s_k; const float* s_v;
  float* v_amax;
  __nv_bfloat16* out;
  int64_t out_ld, q_bs, q_ts;
  int32_t L, Lpad, H, nkb;
  float sc;   // softmax_scale * log2(e)
  // e4m3 output (osb_attn_fp8_blocks): codes of (row, head) at out8 + row * out8_ld + head * 128, scale at
  // out_scale[row * scale_ld + head]
  uint8_t* out8;
  float* out_scale;
  int64_t out8_ld, scale_ld;
};

__global__ void __launch_bounds__(128) attn_fp8_prep_kernel(const Fp8AttnPrep p) {
  __shared__ float s_amax[4][kF8D];
  const int tid = threadIdx.x;
  const int bh = blockIdx.y, b = bh / p.H, h = bh - b * p.H;
  const int t0 = blockIdx.x * 64;
  pdl_wait();   // q, k, v were written by the previous kernel
  {   // ---- one q (threads 0..63) or k (64..127) row: stage, quantize per row ----
    const int kind = tid >> 6, t = t0 + (tid & 63);
    const bool ok = t < p.L;
    const int64_t row = ok ? (int64_t)b * (kind ? p.k_bs : p.q_bs) + (int64_t)t * (kind ? p.k_ts : p.q_ts) : 0;
    const uint4* src = reinterpret_cast<const uint4*>((kind ? p.k : p.q) + row * (kind ? p.k_ld : p.q_ld) + (int64_t)h * kF8D);
    uint4 raw[kF8D / 8];
#pragma unroll
    for (int u = 0; u < kF8D / 8; ++u) raw[u] = ok ? __ldg(src + u) : make_uint4(0, 0, 0, 0);
    const __nv_bfloat16* w1 = kind ? p.kw : p.qw;
    const __nv_bfloat16* w2 = kind ? p.kw2 : p.qw2;
    const __nv_bfloat16* w = (w2 != nullptr && t >= p.norm_split) ? w2 : w1;
    const bool rope = ok && p.cos != nullptr;
    norm_rope_row<kF8D, kF8D / 8>(raw, ok && w1 != nullptr, p.eps, w, rope ? p.cos + (int64_t)t * (kF8D / 2) : nullptr,
                                  rope ? p.sin + (int64_t)t * (kF8D / 2) : nullptr, p.rope_half != 0);
    float amax = 0.f;
#pragma unroll
    for (int u = 0; u < kF8D / 8; ++u) {
      float x[8];
      unpack8(raw[u], x);
#pragma unroll
      for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(x[e]));
    }
    const float s = amax > 0.f ? amax / 448.0f : 1.0f;   // rows t >= L: zero codes, scale 1
    const int64_t r8 = (int64_t)bh * p.Lpad + t;
    uint4* dst = reinterpret_cast<uint4*>((kind ? p.k8 : p.q8) + r8 * kF8D);
#pragma unroll
    for (int u = 0; u < kF8D / 16; ++u) {
      float x[16];
      unpack8(raw[2 * u], x);
      unpack8(raw[2 * u + 1], x + 8);
      dst[u] = e4m3x16(x, s);
    }
    (kind ? p.s_k : p.s_q)[r8] = s;
  }
  {   // ---- v: per-channel amax of the CTA's 64 tokens; thread = (channel unit tid % 16, rows tid / 16 + 8 i) ----
    const int u = tid & 15, r0 = tid >> 4;
    float m[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int t = t0 + r0 + 8 * i;
      if (t < p.L) {
        float x[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.v + ((int64_t)b * p.k_bs + (int64_t)t * p.k_ts) * p.v_ld +
                                                     (int64_t)h * kF8D) + u), x);
#pragma unroll
        for (int e = 0; e < 8; ++e) m[e] = fmaxf(m[e], fabsf(x[e]));
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) m[e] = fmaxf(m[e], __shfl_xor_sync(0xffffffffu, m[e], 16));   // lane l ^ 16: same u
    if ((tid & 31) < 16) {
#pragma unroll
      for (int e = 0; e < 8; ++e) s_amax[tid >> 5][8 * u + e] = m[e];
    }
    __syncthreads();
    const float a = fmaxf(fmaxf(s_amax[0][tid], s_amax[1][tid]), fmaxf(s_amax[2][tid], s_amax[3][tid]));
    if (a > 0.f) atomicMax(reinterpret_cast<unsigned int*>(p.v_amax) + (int64_t)bh * kF8D + tid, __float_as_uint(a));
  }
  pdl_launch_dependents();
}

__global__ void __launch_bounds__(256) attn_fp8_vpack_kernel(const Fp8AttnPrep p) {
  __shared__ __align__(16) __nv_bfloat16 tile[kF8KB][kF8D];   // [key][channel]
  const int tid = threadIdx.x;
  const int bh = blockIdx.y, b = bh / p.H, h = bh - b * p.H;
  const int key0 = blockIdx.x * kF8KB;
  pdl_wait();   // the channel amax of the prep kernel
  for (int i = tid; i < kF8KB * kF8D / 8; i += 256) {
    const int key = i >> 4, u = i & 15, t = key0 + key;
    uint4 x = make_uint4(0, 0, 0, 0);
    if (t < p.L)
      x = __ldg(reinterpret_cast<const uint4*>(p.v + ((int64_t)b * p.k_bs + (int64_t)t * p.k_ts) * p.v_ld +
                                               (int64_t)h * kF8D) + u);
    *reinterpret_cast<uint4*>(&tile[key][8 * u]) = x;
  }
  const int c = tid & 127, half = tid >> 7;
  const float a = p.v_amax[(int64_t)bh * kF8D + c];
  const float s = a > 0.f ? a / 448.0f : 1.0f;
  if (blockIdx.x == 0 && half == 0) p.s_v[(int64_t)bh * kF8D + c] = s;
  __syncthreads();
  uint4* dst = reinterpret_cast<uint4*>(p.vt8 + ((int64_t)bh * kF8D + c) * p.Lpad + key0 + 64 * half);
#pragma unroll
  for (int q = 0; q < 4; ++q) dst[q] = vt8_pack16(tile, c, 64 * half + 16 * q, s);   // pad keys were loaded as zeros
  pdl_launch_dependents();
}

// kOut8: the output leaves as e4m3 codes with one scale per (row, head) instead of bf16
template <bool kOut8>
__global__ void __launch_bounds__(kF8Threads, 1)
attn_fp8_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_vt, const Fp8AttnMain p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw0 = smem_u32(smem_raw);
  const uint32_t base = (raw0 + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 1024-byte aligned
  const uint32_t sQ = base;
  auto sK = [&](int s) { return base + (uint32_t)kF8TileBytes + (uint32_t)s * 2u * kF8TileBytes; };
  auto sV = [&](int s) { return sK(s) + (uint32_t)kF8TileBytes; };
  const uint32_t sScale = base + (uint32_t)kF8TileBytes * (1 + 2 * kF8Stages);
  auto sSk = [&](int s) { return sScale + 512u * s; };
  const uint32_t bar = sScale + 512u * kF8Stages;
  const uint32_t q_full = bar;
  auto full_bar = [&](int s) { return bar + 8u + 8u * s; };
  auto empty_bar = [&](int s) { return bar + 8u + 8u * (kF8Stages + s); };

  const int wg = threadIdx.x >> 7, tid_wg = threadIdx.x & 127;
  const int qt = blockIdx.x, bh = blockIdx.y;
  const int32_t row0 = bh * p.Lpad;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_vt);
    mbar_init(q_full, 1);
    for (int s = 0; s < kF8Stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // the prep and V pack kernels have completed

  if (wg == 0) {
    // ===================== producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
    if (qt == 0) p.v_amax[(int64_t)bh * kF8D + tid_wg] = 0.f;   // read by this call's V pack only: ready for the next call
    if (tid_wg == 0) {
      mbar_expect_tx(q_full, kF8TileBytes);
      tma_load_2d(&tmap_q, q_full, sQ, 0, row0 + qt * kF8KB);
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < p.nkb; ++kb) {
        mbar_wait_notrace(empty_bar(stage), phase ^ 1);
        mbar_expect_tx(full_bar(stage), 2 * kF8TileBytes + 512);
        tma_load_2d(&tmap_k, full_bar(stage), sK(stage), 0, row0 + kb * kF8KB);
        tma_load_2d(&tmap_vt, full_bar(stage), sV(stage), kb * kF8KB, bh * kF8D);
        bulk_load_1d(sSk(stage), p.s_k + row0 + kb * kF8KB, 512, full_bar(stage));
        if (++stage == kF8Stages) { stage = 0; phase ^= 1; }
      }
      pdl_launch_dependents();
    }
    return;
  }

  // ===================== consumers: 64 query rows each =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;\n" ::: "memory");
  const int cw = wg - 1;
  const int lane = tid_wg & 31, quad = lane & 3;
  const int r_loc = cw * 64 + (tid_wg >> 5) * 16 + (lane >> 2);   // rows r_loc and r_loc + 8 of the query tile
  float sq[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) sq[hh] = __ldg(p.s_q + row0 + qt * kF8KB + r_loc + 8 * hh) * p.sc;
  // accumulator fragment: x[4 j + 2 hh + e] = (row r_loc + 8 hh, column 8 j + 2 quad + e)
  float o[64], part[64], s[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = part[i] = s[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const float* sk_gen = reinterpret_cast<const float*>(smem_raw + (sSk(0) - raw0));
  // Every row sees the key slots [0, L) of the 128-key blocks; only the last block is ragged.  Every block holds a
  // valid key, so the running maximum is finite after each block and the guarded alpha of fp8_flash_block is exactly
  // exp2(m - mn).
  const int lo[2] = {0, 0}, hi[2] = {p.L, p.L};

  mbar_wait_notrace(q_full, 0);
  const uint64_t dq = make_sw128_kmajor_desc(sQ + (uint32_t)(cw * 64 * 128));
  int stage = 0;
  uint32_t phase = 0;
  for (int kb = 0; kb < p.nkb; ++kb) {
    mbar_wait_notrace(full_bar(stage), phase);
    fp8_flash_block<kF8D, false>(o, part, s, m, l, dq, sK(stage), sV(stage), sk_gen + 128 * stage, nullptr, sq,
                                 kb * kF8KB, kF8KB, lo, hi, empty_bar(stage));
    if (++stage == kF8Stages) { stage = 0; phase ^= 1; }
  }

  // ---- out = O s_v / (256 l), rows < L ----
  float inv[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    inv[hh] = __fdividef(1.0f, 256.f * l[hh]);   // l >= 1: the row maximum contributes exp2(0)
  }
  const int b = bh / p.H, head = bh - b * p.H;
  const float* sv = p.s_v + (int64_t)bh * kF8D;
  if constexpr (kOut8) {
    // The row's 128 channels (one 1 x 128 scale block) live in the 4 lanes of a quad: block amax by quad shuffles,
    // s = amax / 448 (1 for a zero block), codes e4m3_rn_satfinite(v / s) with IEEE division.
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int i = qt * kF8KB + r_loc + 8 * hh;
      float amax = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 v = __ldg(reinterpret_cast<const float2*>(sv + 8 * j + 2 * quad));
        o[4 * j + 2 * hh] = o[4 * j + 2 * hh] * v.x * inv[hh];
        o[4 * j + 2 * hh + 1] = o[4 * j + 2 * hh + 1] * v.y * inv[hh];
        amax = fmaxf(amax, fmaxf(fabsf(o[4 * j + 2 * hh]), fabsf(o[4 * j + 2 * hh + 1])));
      }
      amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
      amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
      if (i >= p.L) continue;
      const float s = amax > 0.f ? amax / 448.0f : 1.0f;
      const int64_t row = (int64_t)b * p.q_bs + (int64_t)i * p.q_ts;
      uint8_t* dst = p.out8 + row * p.out8_ld + (int64_t)head * kF8D;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<uint16_t*>(dst + 8 * j + 2 * quad) =
            (uint16_t)e4m3x2(o[4 * j + 2 * hh] / s, o[4 * j + 2 * hh + 1] / s);
      if (quad == 0) p.out_scale[row * p.scale_ld + head] = s;
    }
  } else {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int i = qt * kF8KB + r_loc + 8 * hh;
      if (i >= p.L) continue;
      __nv_bfloat16* dst = p.out + ((int64_t)b * p.q_bs + (int64_t)i * p.q_ts) * p.out_ld + (int64_t)head * kF8D;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = 8 * j + 2 * quad;
        const float2 v = __ldg(reinterpret_cast<const float2*>(sv + c));
        *reinterpret_cast<uint32_t*>(dst + c) =
            pack_bf16x2(o[4 * j + 2 * hh] * v.x * inv[hh], o[4 * j + 2 * hh + 1] * v.y * inv[hh]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// osb_head_tiles_fp8 / osb_attn_tiles_fp8
// ---------------------------------------------------------------------------------------------------------------
struct TileFp8Convert {
  const uint8_t* src;
  int64_t kind_stride, head_stride;
  uint8_t* codes;
  float* scales;
  int64_t tiles_per_head;
  int32_t H, TR, v_period, v_slot;
};

template <int D>
__global__ void __launch_bounds__(128) head_tiles_fp8_kernel(const TileFp8Convert p) {
  using Cfg = HeadTileCfg<D>;
  constexpr int U = Cfg::U;
  __shared__ __align__(16) __nv_bfloat16 tile[128][D];   // v only: [tile row][channel]
  const int tid = threadIdx.x;
  const int t = blockIdx.x, head = blockIdx.y, kind = blockIdx.z;
  const uint8_t* src = p.src + (int64_t)kind * p.kind_stride + (int64_t)head * p.head_stride +
                       (int64_t)t * p.TR * Cfg::ROW_BYTES;
  const int64_t ti = ((int64_t)kind * p.H + head) * p.tiles_per_head + t;
  uint8_t* dst = p.codes + ti * kTileF8Bytes;
  float* sdst = p.scales + ti * kTileF8Scales;
  const uint32_t chunk = (uint32_t)p.TR * 128u;
  const bool is_v = p.v_period > 0 && kind % p.v_period == p.v_slot;
  pdl_wait();   // the tiles were written by the previous kernel
  if (!is_v) {   // ---- q / k: row tid ----
    const int r = tid;
    uint4 raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      raw[u] = r < p.TR ? *reinterpret_cast<const uint4*>(src + tile_unit_off<Cfg::MAIN>(r, u, chunk)) : make_uint4(0, 0, 0, 0);
    float amax = 0.f;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float x[8];
      unpack8(raw[u], x);
#pragma unroll
      for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(x[e]));
    }
    const float s = amax > 0.f ? amax / 448.0f : 1.0f;
#pragma unroll
    for (int w = 0; w < 8; ++w) {   // 16 channels per 16-byte unit
      float x[16];
#pragma unroll
      for (int e = 0; e < 16; ++e) x[e] = 0.f;
      if (2 * w < U) unpack8(raw[2 * w], x);
      if (2 * w + 1 < U) unpack8(raw[2 * w + 1], x + 8);
      *reinterpret_cast<uint4*>(dst + r * 128 + ((w ^ (r & 7)) << 4)) = e4m3x16(x, s);
    }
    sdst[r] = s;
  } else {       // ---- v: channel tid ----
    for (int i = tid; i < 128 * U; i += 128) {
      const int r = i / U, u = i - r * U;
      const uint4 x = r < p.TR ? *reinterpret_cast<const uint4*>(src + tile_unit_off<Cfg::MAIN>(r, u, chunk))
                               : make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(&tile[r][8 * u]) = x;
    }
    __syncthreads();
    const int c = tid;
    if (c < D) {
      float amax = 0.f;
      for (int r = 0; r < 128; ++r) amax = fmaxf(amax, fabsf(__bfloat162float(tile[r][c])));
      const float s = amax > 0.f ? amax / 448.0f : 1.0f;
#pragma unroll 1
      for (int w = 0; w < 8; ++w)   // key positions 16 w .. 16 w + 15
        *reinterpret_cast<uint4*>(dst + c * 128 + ((w ^ (c & 7)) << 4)) = vt8_pack16(tile, c, 16 * w, s);
      sdst[c] = s;
    } else {
      sdst[c] = 1.0f;
    }
  }
  pdl_launch_dependents();
}

struct TileFp8Attn {
  const uint8_t* q8; const uint8_t* k8; const uint8_t* v8;
  const float* s_q; const float* s_k; const float* s_v;
  int64_t q_head_tiles, kv_head_tiles;
  float sc;   // softmax_scale * log2(e)
  TileSets ts;
};

template <int D>
__global__ void __launch_bounds__(kF8Threads, 1) attn_tiles_fp8_kernel(const TileFp8Attn p) {
  constexpr int NO = D / 2;               // O / partial accumulator registers per thread (N = D)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw0 = smem_u32(smem_raw);
  const uint32_t base = (raw0 + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 1024-byte aligned
  const uint32_t sQ = base;
  auto sK = [&](int s) { return base + (uint32_t)kTileF8Bytes + (uint32_t)s * kTF8StageBytes; };
  auto sV = [&](int s) { return sK(s) + (uint32_t)kTileF8Bytes; };
  auto sSk = [&](int s) { return sV(s) + (uint32_t)kTileF8Bytes; };
  auto sSv = [&](int s) { return sSk(s) + 512u; };
  const uint32_t bar = base + (uint32_t)kTileF8Bytes + (uint32_t)kTF8Stages * kTF8StageBytes;
  const uint32_t q_full = bar;
  auto full_bar = [&](int s) { return bar + 8u + 8u * s; };
  auto empty_bar = [&](int s) { return bar + 8u + 8u * (kTF8Stages + s); };

  const TileSets& ts = p.ts;
  const int wg = threadIdx.x >> 7, tid_wg = threadIdx.x & 127;
  const int64_t qtile = blockIdx.x;
  const int head = blockIdx.y;
  const int64_t set = qtile / ts.qmap.tps;
  const int qt = (int)(qtile - set * ts.qmap.tps);
  const int keys = tile_set_keys(ts, set);
  const int nkt = (keys + ts.BK - 1) / ts.BK;   // key tiles holding valid keys
  const int64_t qti = (int64_t)head * p.q_head_tiles + qtile;
  const int64_t kti0 = (int64_t)head * p.kv_head_tiles + set * ts.nkb;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < kTF8Stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // the e4m3 tiles were written by the previous kernel

  if (wg == 0) {
    // ===================== producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;\n" ::: "memory");
    if (tid_wg == 0) {
      mbar_expect_tx(q_full, kTileF8Bytes);
      bulk_load_1d(sQ, p.q8 + qti * kTileF8Bytes, kTileF8Bytes, q_full);
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < nkt; ++kb) {
        const int64_t ti = kti0 + kb;
        mbar_wait_notrace(empty_bar(stage), phase ^ 1);
        mbar_expect_tx(full_bar(stage), kTileF8Bytes + D * 128 + 1024);
        bulk_load_1d(sK(stage), p.k8 + ti * kTileF8Bytes, kTileF8Bytes, full_bar(stage));
        bulk_load_1d(sV(stage), p.v8 + ti * kTileF8Bytes, D * 128, full_bar(stage));
        bulk_load_1d(sSk(stage), p.s_k + ti * kTileF8Scales, 512, full_bar(stage));
        bulk_load_1d(sSv(stage), p.s_v + ti * kTileF8Scales, 512, full_bar(stage));
        if (++stage == kTF8Stages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================== consumers: 64 query rows each =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;\n" ::: "memory");
  const int cw = wg - 1;
  const int lane = tid_wg & 31, quad = lane & 3;
  const int r_loc = cw * 64 + (tid_wg >> 5) * 16 + (lane >> 2);   // rows r_loc and r_loc + 8 of the query tile
  // my two query rows: sequence, position, valid key range [lo, hi) in the set's key slots
  int64_t seq[2];
  int pos[2], lo[2], hi[2];
  bool valid[2];
  float sq[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = r_loc + 8 * hh;
    tile_query_row(ts, set, qt, keys, r, seq[hh], pos[hh], valid[hh], lo[hh], hi[hh]);
    sq[hh] = __ldg(p.s_q + qti * kTileF8Scales + r) * p.sc;
  }
  // accumulator fragment: x[4 j + 2 hh + e] = (row r_loc + 8 hh, column 8 j + 2 quad + e)
  float o[NO], part[NO], s[64];
#pragma unroll
  for (int i = 0; i < NO; ++i) o[i] = part[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 64; ++i) s[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const float* sk_gen = reinterpret_cast<const float*>(smem_raw + (sSk(0) - raw0));
  const float* sv_gen = reinterpret_cast<const float*>(smem_raw + (sSv(0) - raw0));

  mbar_wait_notrace(q_full, 0);
  const uint64_t dq = make_sw128_kmajor_desc(sQ + (uint32_t)(cw * 64 * 128));
  int stage = 0;
  uint32_t phase = 0;
  for (int kb = 0; kb < nkt; ++kb) {
    mbar_wait_notrace(full_bar(stage), phase);
    fp8_flash_block<D, true>(o, part, s, m, l, dq, sK(stage), sV(stage), sk_gen + (kTF8StageBytes / 4) * stage,
                             sv_gen + (kTF8StageBytes / 4) * stage, sq, kb * ts.BK, ts.BK, lo, hi, empty_bar(stage));
    if (++stage == kTF8Stages) { stage = 0; phase ^= 1; }
  }
  pdl_launch_dependents();

  // ---- out = O / (256 l) ----
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float lt = l[hh];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const float inv = lt > 0.f ? __fdividef(1.0f, 256.f * lt) : 0.f;   // no valid key: zeros
    if (!valid[hh]) continue;
    __nv_bfloat16* dst = tile_out_row(ts, seq[hh], pos[hh]) + (int64_t)head * D;
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j + 2 * quad) = pack_bf16x2(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
  }
}

int attn_fp8_init() {
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_fp8_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kF8Smem));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_fp8_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kF8Smem));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_fp8_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTF8Smem));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_fp8_kernel<72>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTF8Smem));
  return OSB_OK;
}

}  // namespace osb

namespace osb {
namespace {

// osb_attn_fp8 (o8 == nullptr: bf16 out) and osb_attn_fp8_blocks (e4m3 codes + block scales through o8)
int attn_fp8_launch(const osb_attn_short_args* a, const osb_attn_fp8_workspace* ws, const osb_attn_fp8_out* o8,
                    void* stream, const char* who) {
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  osb_attn_short_args chk;
  if (o8 != nullptr) {   // the codes take the place of out in the argument checks
    OSB_REQUIRE(a != nullptr, "%s: null args", who);
    OSB_REQUIRE(o8->codes && o8->scales, "%s: null output codes or scales", who);
    OSB_REQUIRE((reinterpret_cast<uintptr_t>(o8->scales) & 3) == 0 && o8->scales_ld >= a->num_heads,
                "%s: scales must be 4-byte aligned with a row stride >= num_heads (%lld < %d)", who,
                (long long)o8->scales_ld, a->num_heads);
    chk = *a;
    chk.out = o8->codes;
    chk.out_ld = o8->codes_ld;
    a = &chk;
  }
  const int rc0 = check_attn_short_args(a, who);
  if (rc0) return rc0;
  OSB_REQUIRE(ws != nullptr, "%s: null workspace", who);
  OSB_REQUIRE(a->head_dim == kF8D, "%s: head_dim %d not built (128)", who, a->head_dim);
  OSB_REQUIRE(a->Lq == a->Lk, "%s: self-attention only (Lq %d != Lk %d)", who, a->Lq, a->Lk);
  OSB_REQUIRE(a->kv_lens == nullptr, "%s: kv_lens is not supported", who);
  OSB_REQUIRE(a->seqs_per_batch == 1, "%s: one sequence per batch element (seqs_per_batch %lld)", who,
              (long long)a->seqs_per_batch);
  const int64_t BH = a->num_seqs * a->num_heads;
  const int32_t L = a->Lq, Lpad = (L + kF8KB - 1) / kF8KB * kF8KB;
  OSB_REQUIRE(ws->q8 && ws->k8 && ws->vt8 && ws->s_q && ws->s_k && ws->s_v && ws->v_amax, "%s: null workspace buffer", who);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(ws->q8) | reinterpret_cast<uintptr_t>(ws->k8) | reinterpret_cast<uintptr_t>(ws->vt8) |
                reinterpret_cast<uintptr_t>(ws->s_q) | reinterpret_cast<uintptr_t>(ws->s_k) | reinterpret_cast<uintptr_t>(ws->s_v) |
                reinterpret_cast<uintptr_t>(ws->v_amax)) & 15) == 0, "%s: workspace buffers must be 16-byte aligned", who);
  OSB_REQUIRE(BH <= ws->capacity_bh && Lpad <= ws->capacity_lpad,
              "%s: workspace for %lld x %lld holds less than %lld sequence-heads x %d padded tokens",
              who, (long long)ws->capacity_bh, (long long)ws->capacity_lpad, (long long)BH, Lpad);
  OSB_REQUIRE(BH <= 65535 && BH * Lpad < (1ll << 31), "%s: problem too large (%lld sequence-heads of %d)", who,
              (long long)BH, Lpad);

  Fp8AttnPrep pp = {};
  pp.q = static_cast<const __nv_bfloat16*>(a->q);
  pp.k = static_cast<const __nv_bfloat16*>(a->k);
  pp.v = static_cast<const __nv_bfloat16*>(a->v);
  pp.q_ld = a->q_ld; pp.k_ld = a->k_ld; pp.v_ld = a->v_ld;
  pp.q_bs = a->q_batch_stride; pp.q_ts = a->q_tok_stride;
  pp.k_bs = a->k_batch_stride; pp.k_ts = a->k_tok_stride;
  pp.L = L; pp.Lpad = Lpad; pp.H = a->num_heads;
  pp.qw = static_cast<const __nv_bfloat16*>(a->q_norm_w);
  pp.kw = static_cast<const __nv_bfloat16*>(a->k_norm_w);
  pp.qw2 = static_cast<const __nv_bfloat16*>(a->q_norm_w2);
  pp.kw2 = static_cast<const __nv_bfloat16*>(a->k_norm_w2);
  pp.norm_split = a->norm_split;
  pp.eps = a->norm_eps;
  pp.cos = a->rope_cos; pp.sin = a->rope_sin;
  pp.rope_half = a->rope_cos != nullptr && a->rope_half ? 1 : 0;
  pp.q8 = static_cast<uint8_t*>(ws->q8); pp.k8 = static_cast<uint8_t*>(ws->k8); pp.vt8 = static_cast<uint8_t*>(ws->vt8);
  pp.s_q = ws->s_q; pp.s_k = ws->s_k; pp.s_v = ws->s_v; pp.v_amax = ws->v_amax;

  CUtensorMap tq, tk, tv;
  int rc = make_tmap_2d_e4m3(&tq, ws->q8, (uint64_t)BH * Lpad, kF8D, kF8D, kF8KB, kF8D);
  if (rc) return rc;
  rc = make_tmap_2d_e4m3(&tk, ws->k8, (uint64_t)BH * Lpad, kF8D, kF8D, kF8KB, kF8D);
  if (rc) return rc;
  rc = make_tmap_2d_e4m3(&tv, ws->vt8, (uint64_t)BH * kF8D, Lpad, Lpad, kF8D, kF8KB);
  if (rc) return rc;

  Fp8AttnMain pm = {};
  pm.s_q = ws->s_q; pm.s_k = ws->s_k; pm.s_v = ws->s_v; pm.v_amax = ws->v_amax;
  pm.out = static_cast<__nv_bfloat16*>(a->out);
  pm.out_ld = a->out_ld; pm.q_bs = a->q_batch_stride; pm.q_ts = a->q_tok_stride;
  pm.L = L; pm.Lpad = Lpad; pm.H = a->num_heads; pm.nkb = Lpad / kF8KB;
  pm.sc = a->softmax_scale * 1.4426950408889634f;
  if (o8 != nullptr) {
    pm.out = nullptr;
    pm.out8 = static_cast<uint8_t*>(o8->codes);
    pm.out_scale = o8->scales;
    pm.out8_ld = o8->codes_ld;
    pm.scale_ld = o8->scales_ld;
  }

  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)(Lpad / 64), (unsigned)BH), dim3(128), 0, s, attr);
  OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_fp8_prep_kernel, pp));
  cfg = launch_config(dim3((unsigned)(Lpad / kF8KB), (unsigned)BH), dim3(256), 0, s, attr);
  OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_fp8_vpack_kernel, pp));
  cfg = launch_config(dim3((unsigned)(Lpad / kF8KB), (unsigned)BH), dim3(kF8Threads), kF8Smem, s, attr);
  if (o8 != nullptr) { OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_fp8_kernel<true>, tq, tk, tv, pm)); }
  else { OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_fp8_kernel<false>, tq, tk, tv, pm)); }
  count_launch(3);
  return OSB_OK;
}

}  // namespace
}  // namespace osb

extern "C" int osb_attn_fp8(const osb_attn_short_args* a, const osb_attn_fp8_workspace* ws, void* stream) {
  return osb::attn_fp8_launch(a, ws, nullptr, stream, "osb_attn_fp8");
}

extern "C" int osb_attn_fp8_blocks(const osb_attn_short_args* a, const osb_attn_fp8_workspace* ws,
                                   const osb_attn_fp8_out* out, void* stream) {
  using namespace osb;
  OSB_REQUIRE(out != nullptr, "osb_attn_fp8_blocks: null output args");
  return attn_fp8_launch(a, ws, out, stream, "osb_attn_fp8_blocks");
}

extern "C" int osb_head_tiles_fp8(const osb_head_tiles_fp8_args* a, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(a != nullptr, "osb_head_tiles_fp8: null args");
  OSB_REQUIRE(a->tiles && a->dst.codes && a->dst.scales, "osb_head_tiles_fp8: null tensor");
  const int D = a->head_dim;
  OSB_REQUIRE(D == 64 || D == 72, "osb_head_tiles_fp8: head_dim %d not built (64, 72)", D);
  OSB_REQUIRE(a->tile_rows > 0 && a->tile_rows <= 128 && a->tile_rows % 8 == 0,
              "osb_head_tiles_fp8: tile_rows must be 8..128 in multiples of 8, got %d", a->tile_rows);
  OSB_REQUIRE(a->nkinds >= 1 && a->nkinds <= 65535 && a->dst.num_heads >= 1 && a->dst.num_heads <= 65535 &&
              a->dst.tiles_per_head >= 1 && a->dst.tiles_per_head < (1ll << 31),
              "osb_head_tiles_fp8: empty or too large (%d kinds, %d heads, %lld tiles per head)", a->nkinds,
              a->dst.num_heads, (long long)a->dst.tiles_per_head);
  OSB_REQUIRE(a->v_period >= 0 && (a->v_period == 0 || (a->v_slot >= 0 && a->v_slot < a->v_period)),
              "osb_head_tiles_fp8: bad value-kind rule (period %d slot %d)", a->v_period, a->v_slot);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(a->tiles) | reinterpret_cast<uintptr_t>(a->dst.codes) |
                reinterpret_cast<uintptr_t>(a->dst.scales)) & 15) == 0 && a->kind_stride % 16 == 0 && a->head_stride % 16 == 0,
              "osb_head_tiles_fp8: buffers must be 16-byte aligned");
  TileFp8Convert p = {};
  p.src = static_cast<const uint8_t*>(a->tiles);
  p.kind_stride = a->kind_stride; p.head_stride = a->head_stride;
  p.codes = static_cast<uint8_t*>(a->dst.codes);
  p.scales = a->dst.scales;
  p.tiles_per_head = a->dst.tiles_per_head;
  p.H = a->dst.num_heads; p.TR = a->tile_rows; p.v_period = a->v_period; p.v_slot = a->v_slot;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)p.tiles_per_head, (unsigned)p.H, (unsigned)a->nkinds), dim3(128), 0,
                                         s, attr);
  if (D == 64) { OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, head_tiles_fp8_kernel<64>, p)); }
  else { OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, head_tiles_fp8_kernel<72>, p)); }
  count_launch();
  return OSB_OK;
}

extern "C" int osb_attn_tiles_fp8(const osb_attn_tiles_args* a, const osb_attn_tiles_fp8_operands* ops, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(a != nullptr && ops != nullptr, "osb_attn_tiles_fp8: null args");
  OSB_REQUIRE(ops->q8 && ops->k8 && ops->v8 && ops->s_q && ops->s_k && ops->s_v, "osb_attn_tiles_fp8: null tensor");
  const int D = a->head_dim;
  OSB_REQUIRE(D == 64 || D == 72, "osb_attn_tiles_fp8: head_dim %d not built (64, 72)", D);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(ops->q8) | reinterpret_cast<uintptr_t>(ops->k8) | reinterpret_cast<uintptr_t>(ops->v8) |
                reinterpret_cast<uintptr_t>(ops->s_q) | reinterpret_cast<uintptr_t>(ops->s_k) |
                reinterpret_cast<uintptr_t>(ops->s_v)) & 15) == 0,
              "osb_attn_tiles_fp8: e4m3 tiles and scales must be 16-byte aligned");
  TileFp8Attn p = {};
  const int rc = make_tile_sets(&p.ts, a, "osb_attn_tiles_fp8");
  if (rc) return rc;
  OSB_REQUIRE(a->num_heads <= 65535, "osb_attn_tiles_fp8: %d heads (at most 65535)", a->num_heads);
  const int64_t qtiles = p.ts.num_sets * p.ts.qmap.tps;
  OSB_REQUIRE(ops->q_head_tiles >= qtiles && ops->kv_head_tiles >= p.ts.num_sets * a->kv_tiles_per_set,
              "osb_attn_tiles_fp8: %lld / %lld tiles per head hold less than %lld query / %lld key tiles",
              (long long)ops->q_head_tiles, (long long)ops->kv_head_tiles, (long long)qtiles,
              (long long)(p.ts.num_sets * a->kv_tiles_per_set));
  OSB_REQUIRE(qtiles < (1ll << 31), "osb_attn_tiles_fp8: problem too large (%lld query tiles)", (long long)qtiles);
  p.q8 = static_cast<const uint8_t*>(ops->q8);
  p.k8 = static_cast<const uint8_t*>(ops->k8);
  p.v8 = static_cast<const uint8_t*>(ops->v8);
  p.s_q = ops->s_q; p.s_k = ops->s_k; p.s_v = ops->s_v;
  p.q_head_tiles = ops->q_head_tiles; p.kv_head_tiles = ops->kv_head_tiles;
  p.sc = a->softmax_scale * 1.4426950408889634f;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)qtiles, (unsigned)a->num_heads), dim3(kF8Threads), kTF8Smem, s, attr);
  if (D == 64) { OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_tiles_fp8_kernel<64>, p)); }
  else { OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_tiles_fp8_kernel<72>, p)); }
  count_launch();
  return OSB_OK;
}
