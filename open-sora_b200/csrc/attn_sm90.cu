// Attention on sm_90a: softmax(q k^T * scale) v per (sequence, head), non-causal, exact online softmax.
//
// Key / value tiles sit in shared memory in the head-tile layout (tiles.cuh: 64-column chunks with the 128-byte swizzle
// plus the head-dim tail).  P is rounded to bf16 straight from the S accumulator registers, which already have the
// layout of the A operand of the PV product, so S and P never touch shared memory.
//
//   osb_attn_tiles: q / k / v arrive as operand-tile images written by the projection GEMM's head-tile epilogue
//                   (bias, RMSNorm and RoPE applied there).  attn_tiles_kernel is persistent and warp-specialized: a
//                   producer warpgroup bulk-copies Q tiles and a ring of K / V tiles (kept resident while consecutive
//                   work items share them) and two consumer warpgroups run S = Q K^T and O += P V on wgmma, reading the
//                   tile images as shared-memory descriptors.
//   osb_attn_short: the flash core below.  One CTA (8 warps) owns 128 query rows of one head; every warp owns 16 rows
//                   and keeps its Q fragments, the running row maximum / sum and the fp32 O accumulator in registers;
//                   the 16-byte rows that ldmatrix gathers are bank-conflict free for K and for V read transposed, and
//                   the tensor core work is mma.sync m16n8k16 (bf16 in, fp32 accumulate).
//                   q / k / v are token-layout rows (any strides); the CTA stages them into the same tile layout,
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
#include "stage.cuh"
#include "tiles.cuh"
#include "wgmma.cuh"

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
  int32_t q_tile_bytes, kv_tile_bytes;                    // TRq * ROW_BYTES, BK * ROW_BYTES
  int64_t items;                                          // heads x sets x query tiles per set
  float scale_log2;
  TileSets ts;
};

// Shared-memory carve-up of attn_tiles_kernel<D>: two Q slots and a ring of K / V stages, every slot sized for 128 rows
// whatever the tile rows are (the wgmma products read 64 query rows per consumer and 128 key rows per tile), then the
// mbarriers.  One CTA per SM: the carve-up is more than half of the 227 KB an SM offers.
template <int D>
struct TileAttnSmem {
  static constexpr int kSlot = 128 * HeadTileCfg<D>::ROW_BYTES;   // 1024-byte multiple
  static constexpr int kStages = D == 128 ? 2 : (D == 72 ? 4 : 5);
  static constexpr int kData = 2 * kSlot + kStages * 2 * kSlot;
  static constexpr int kBytes = 1024 + kData + 8 * (4 + 2 * kStages);   // + alignment slack
  static_assert(kBytes <= 227 * 1024 && 2 * kBytes > 228 * 1024, "one resident CTA per SM");
};

constexpr int kTileAttnThreads = 384;   // producer warpgroup + two consumer warpgroups of 64 query rows

// Persistent: CTA b owns the work items [b * items / grid, (b + 1) * items / grid), item = (head * sets + set) * tps + q
// tile, so consecutive items mostly share a (head, set).  Warpgroup 0 (one thread) bulk-copies each item's Q tile into
// one of two slots and its key / value tiles into the stage ring while the consumers work on the item before; when an
// item has the (head, set) of the item before and the set's key tiles fit the ring, they are still resident and are
// not loaded again.  Warpgroups 1 and 2 own 64 query rows each: S = Q K^T on wgmma (both operands shared-memory
// descriptors over the tile images), masks and the exact online softmax over one 128-key tile at a time in registers,
// P rounded to bf16 into the register A fragment of O += P V (V read MN-major from the same tile image).  A stage is
// released once the PV product that read it retired, unless the next item reuses it.
template <int D>
__global__ void __launch_bounds__(kTileAttnThreads, 1) attn_tiles_kernel(const TileAttnParams p) {
  using Cfg = HeadTileCfg<D>;
  using Sm = TileAttnSmem<D>;
  constexpr int MAIN = Cfg::MAIN, TAIL = Cfg::TAIL, STAGES = Sm::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 1024-byte aligned
  auto sQ = [&](int b) { return base + (uint32_t)(b * Sm::kSlot); };
  auto sK = [&](int s) { return base + (uint32_t)((2 + 2 * s) * Sm::kSlot); };
  auto sV = [&](int s) { return sK(s) + (uint32_t)Sm::kSlot; };
  const uint32_t bar = base + (uint32_t)Sm::kData;
  auto q_full = [&](int b) { return bar + 8u * b; };
  auto q_empty = [&](int b) { return bar + 16u + 8u * b; };
  auto full_bar = [&](int s) { return bar + 32u + 8u * s; };
  auto empty_bar = [&](int s) { return bar + 32u + 8u * (STAGES + s); };

  const int wg = threadIdx.x >> 7, tid_wg = threadIdx.x & 127;
  const int64_t begin = (int64_t)blockIdx.x * p.items / gridDim.x, end = (int64_t)(blockIdx.x + 1) * p.items / gridDim.x;
  const TileSets& ts = p.ts;
  const int tps = ts.qmap.tps;

  // Rows past a tile's rows are read by the products (key rows up to 128 for every tile, query rows up to 64 per
  // consumer) and must be finite: P = 0 times a NaN left in shared memory would still be a NaN.
  {
    uint4* z = reinterpret_cast<uint4*>(smem_raw + (base - smem_u32(smem_raw)));
    for (int i = threadIdx.x; i < Sm::kData / 16; i += kTileAttnThreads) z[i] = make_uint4(0, 0, 0, 0);
  }
  fence_proxy_async_smem();   // the zeros are ordered before the bulk copies into the same bytes
  if (threadIdx.x == 0) {
    for (int b = 0; b < 2; ++b) { mbar_init(q_full(b), 1); mbar_init(q_empty(b), 2); }
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }   // 2: one per consumer
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // the tiles were written by the previous kernel, which may also still read `out`

  if (wg == 0) {
    // ===================== producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (tid_wg == 0) {
      uint32_t kv_it = 0;   // K / V tile loads so far: stage kv_it % STAGES, ring pass kv_it / STAGES
      for (int64_t it = begin; it < end; ++it) {
        const uint32_t n = (uint32_t)(it - begin);
        const int64_t hs = it / tps, head = hs / ts.num_sets, set = hs - head * ts.num_sets;
        const int qs = n & 1;
        mbar_wait_notrace(q_empty(qs), ((n >> 1) & 1u) ^ 1u);
        mbar_expect_tx(q_full(qs), (uint32_t)p.q_tile_bytes);
        bulk_load_1d(sQ(qs), p.q + head * p.q_head_stride + (it - head * ts.num_sets * tps) * p.q_tile_bytes,
                     (uint32_t)p.q_tile_bytes, q_full(qs));
        const int nkt = (tile_set_keys(ts, set) + ts.BK - 1) / ts.BK;
        if (it > begin && (it - 1) / tps == hs && nkt <= STAGES) continue;   // the set's key tiles are resident
        const int64_t off = head * p.kv_head_stride + set * ts.nkb * (int64_t)p.kv_tile_bytes;
        for (int t = 0; t < nkt; ++t, ++kv_it) {
          const int s = (int)(kv_it % STAGES);
          mbar_wait_notrace(empty_bar(s), ((kv_it / STAGES) & 1u) ^ 1u);
          mbar_expect_tx(full_bar(s), 2u * (uint32_t)p.kv_tile_bytes);
          bulk_load_1d(sK(s), p.k + off + (int64_t)t * p.kv_tile_bytes, (uint32_t)p.kv_tile_bytes, full_bar(s));
          bulk_load_1d(sV(s), p.v + off + (int64_t)t * p.kv_tile_bytes, (uint32_t)p.kv_tile_bytes, full_bar(s));
        }
      }
      pdl_launch_dependents();   // every load of this CTA is issued
    }
    return;
  }

  // ===================== consumers: 64 query rows each =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int cw = wg - 1;
  const int lane = tid_wg & 31, quad = lane & 3;
  const int r_loc = cw * 64 + (tid_wg >> 5) * 16 + (lane >> 2);   // rows r_loc and r_loc + 8 of the query tile
  const float sc = p.scale_log2;
  // accumulator fragments: x[4 j + 2 hh + e] = (row r_loc + 8 hh, column 8 j + 2 quad + e)
  float s[64], o[MAIN][32], ot[TAIL ? 8 : 1];
#pragma unroll
  for (int i = 0; i < 64; ++i) s[i] = 0.f;
  uint32_t kv_it = 0, kv0 = 0;   // the producer's count of K / V tile loads; kv0: first load of the current set
  for (int64_t it = begin; it < end; ++it) {
    const uint32_t n = (uint32_t)(it - begin);
    const int64_t hs = it / tps, head = hs / ts.num_sets, set = hs - head * ts.num_sets;
    const int qt = (int)(it - hs * tps), qs = n & 1;
    const int keys = tile_set_keys(ts, set);
    const int nkt = (keys + ts.BK - 1) / ts.BK;
    if (!(it > begin && (it - 1) / tps == hs && nkt <= STAGES)) { kv0 = kv_it; kv_it += nkt; }
    const bool keep = it + 1 < end && (it + 1) / tps == hs && nkt <= STAGES;   // the next item reads these stages

    // my two query rows: sequence, position, valid key range [lo, hi) in the set's key slots
    int64_t seq[2];
    int pos[2], lo[2], hi[2];
    bool valid[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) tile_query_row(ts, set, qt, keys, r_loc + 8 * hh, seq[hh], pos[hh], valid[hh], lo[hh], hi[hh]);
#pragma unroll
    for (int c = 0; c < MAIN; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
#pragma unroll
    for (int i = 0; i < (TAIL ? 8 : 1); ++i) ot[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};

    // Q rows [64 cw, 64 cw + 64) of the slot; 64-column chunks TR * 128 bytes apart, then the tail
    const uint32_t q_chunk = (uint32_t)ts.qmap.TR * 128u, kv_chunk = (uint32_t)ts.BK * 128u;
    const uint32_t qa = sQ(qs) + (uint32_t)(cw * 64 * 128), qa_tail = sQ(qs) + MAIN * q_chunk + (uint32_t)(cw * 8 * 256);
    mbar_wait_notrace(q_full(qs), (n >> 1) & 1u);
    for (int t = 0; t < nkt; ++t) {
      const uint32_t u = kv0 + (uint32_t)t;
      const int st = (int)(u % STAGES);
      mbar_wait_notrace(full_bar(st), (u / STAGES) & 1u);
      // ---- S = Q K^T over 128 key rows (rows past BK are masked) ----
      const uint32_t ka = sK(st), va = sV(st);
      wgmma_fence_regs(s);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < MAIN; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          Wgmma<128>::mma(s, make_sw128_kmajor_desc(qa + c * q_chunk + 32u * k),
                          make_sw128_kmajor_desc(ka + c * kv_chunk + 32u * k), (c | k) ? 1u : 0u);
      if constexpr (TAIL != 0)
        Wgmma<128>::mma(s, make_noswizzle_desc(qa_tail, 128u, 256u), make_noswizzle_desc(ka + MAIN * kv_chunk, 128u, 256u), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      if (t == nkt - 1 && tid_wg == 0) mbar_arrive(q_empty(qs));   // the item's last read of its Q slot retired
      // ---- mask, tile maximum ----
      const int slot0 = t * ts.BK;
      // 16-key groups of the tile before the set's last valid key (>= 1): later groups have P = 0 in every row, so
      // their exp2 is skipped (the text keys of a cross-attention end 4 keys into their third tile).  Their PV k steps
      // still run: a branch around them would make ptxas serialise every wgmma of the kernel (C7520).
      const int n16 = ((keys - slot0 < ts.BK ? keys - slot0 : ts.BK) + 15) >> 4;
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int hh = (i >> 1) & 1;
        const int col = 8 * (i >> 2) + 2 * quad + (i & 1), key = slot0 + col;
        if (col >= ts.BK || key < lo[hh] || key >= hi[hh]) s[i] = -INFINITY;
        mx[hh] = fmaxf(mx[hh], s[i]);
      }
      float alpha[2], ms[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
        const float mn = fmaxf(m[hh], mx[hh]);
        alpha[hh] = (mn == -INFINITY) ? 1.f : fast_exp2((m[hh] - mn) * sc);   // m == -inf: exp2(-inf) = 0
        ms[hh] = (mn == -INFINITY) ? 0.f : mn * sc;
        m[hh] = mn;
        l[hh] *= alpha[hh];
      }
#pragma unroll
      for (int c = 0; c < MAIN; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[c][i] *= alpha[(i >> 1) & 1];
      if constexpr (TAIL != 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) ot[i] *= alpha[(i >> 1) & 1];
      }
      // ---- P = exp2(S * sc - max) (masked scores are -inf and give 0), bf16 A fragments of the 8 k16 steps ----
      uint32_t pa[8][4];
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        s[i] = (i >> 3) < n16 ? fast_exp2(fmaf(s[i], sc, -ms[(i >> 1) & 1])) : 0.f;
        l[(i >> 1) & 1] += s[i];
      }
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        pa[g][0] = pack_bf16x2(s[8 * g + 0], s[8 * g + 1]);
        pa[g][1] = pack_bf16x2(s[8 * g + 2], s[8 * g + 3]);
        pa[g][2] = pack_bf16x2(s[8 * g + 4], s[8 * g + 5]);
        pa[g][3] = pack_bf16x2(s[8 * g + 6], s[8 * g + 7]);
      }
      // ---- O += P V: V MN-major, 16 keys per k step = two 8-row swizzle atoms (2048 B) / tail groups (512 B) ----
#pragma unroll
      for (int c = 0; c < MAIN; ++c) wgmma_fence_regs(o[c]);
      if constexpr (TAIL != 0) wgmma_fence_regs(ot);
      wgmma_fence();
#pragma unroll
      for (int g = 0; g < 8; ++g) {
#pragma unroll
        for (int c = 0; c < MAIN; ++c)
          WgmmaRegAT<64>::mma(o[c], pa[g], make_sw128_kmajor_desc(va + c * kv_chunk + 2048u * g), 1u);
        if constexpr (TAIL != 0)
          WgmmaRegAT<16>::mma(ot, pa[g], make_noswizzle_desc(va + MAIN * kv_chunk + 512u * g, 256u, 128u), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < MAIN; ++c) wgmma_fence_regs(o[c]);
      if constexpr (TAIL != 0) wgmma_fence_regs(ot);
#pragma unroll
      for (int g = 0; g < 8; ++g) fence_regs_u32(pa[g]);   // the A registers stay untouched until the product retired
      if (!keep && tid_wg == 0) mbar_arrive(empty_bar(st));
    }
    if (nkt == 0 && tid_wg == 0) mbar_arrive(q_empty(qs));

    // ---- normalise, round once to bf16, store through the inverse q map ----
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float lt = l[hh];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const float inv = lt > 0.f ? 1.0f / lt : 0.f;   // no valid key: zeros, never 0 * garbage
      if (!valid[hh]) continue;
      __nv_bfloat16* dst = tile_out_row(ts, seq[hh], pos[hh]) + head * D + 2 * quad;
#pragma unroll
      for (int c = 0; c < MAIN; ++c)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint32_t*>(dst + 64 * c + 8 * j) = pack_bf16x2(o[c][4 * j + 2 * hh] * inv, o[c][4 * j + 2 * hh + 1] * inv);
      if constexpr (TAIL != 0)   // columns 64 MAIN .. + 7 (the rest of the tail is padding)
        *reinterpret_cast<uint32_t*>(dst + 64 * MAIN) = pack_bf16x2(ot[2 * hh] * inv, ot[2 * hh + 1] * inv);
    }
  }
}

template <int D>
static int attn_tiles_launch(TileAttnParams& p, int H, cudaStream_t stream) {
  using Cfg = HeadTileCfg<D>;
  p.q_tile_bytes = p.ts.qmap.TR * Cfg::ROW_BYTES;
  p.kv_tile_bytes = p.ts.BK * Cfg::ROW_BYTES;
  p.items = (int64_t)H * p.ts.num_sets * p.ts.qmap.tps;
  if (p.items >= (1ll << 31)) { set_error("osb_attn_tiles: problem too large (%lld work items)", (long long)p.items); return OSB_ERR_UNSUPPORTED; }
  const int64_t grid = p.items < sm_count() ? p.items : sm_count();   // every CTA resident at once
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)grid), dim3(kTileAttnThreads), TileAttnSmem<D>::kBytes, stream, attr);
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

// One head row (U raw bf16x8 units) -> optional RMSNorm scale r*w and RoPE in fp32 -> bf16 (stage.cuh) -> row `row` of
// a tile image in shared memory (64-column chunks chunk_bytes apart, head-dim tail zero padded).
template <int D>
__device__ __forceinline__ void stage_row(uint4 (&raw)[HeadTileCfg<D>::U], bool norm, float eps, const __nv_bfloat16* w,
                                          const float* cosr, const float* sinr, bool rope_half, uint8_t* tile,
                                          uint32_t chunk_bytes, int row) {
  using Cfg = HeadTileCfg<D>;
  constexpr int U = Cfg::U;
  norm_rope_row<D, U>(raw, norm, eps, w, cosr, sinr, rope_half);
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
  constexpr int kMax = 200 * 1024;   // attn_short: a 128-row Q tile and a 64-row K / V block (64 KB at D = 128)
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_short_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_short_kernel<72, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_short_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_short_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMax));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, TileAttnSmem<64>::kBytes));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_kernel<72>, cudaFuncAttributeMaxDynamicSharedMemorySize, TileAttnSmem<72>::kBytes));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, TileAttnSmem<128>::kBytes));
  return OSB_OK;
}

int make_tile_map(TileMap* dst, const osb_tile_map& m, const char* who) {
  OSB_REQUIRE(m.mode == 0 || m.mode == 1, "%s: unknown tile map mode %d", who, m.mode);
  OSB_REQUIRE(m.L > 0 && m.G >= 1 && m.tile_rows > 0 && m.tile_rows <= 128 && m.tile_rows % 8 == 0,
              "%s: bad tile map (L %d G %d rows %d)", who, m.L, m.G, m.tile_rows);
  OSB_REQUIRE(m.G == 1 ? (m.tps == (m.L + m.tile_rows - 1) / m.tile_rows) : (m.G * m.L <= m.tile_rows && m.tps == 1),
              "%s: tile map inconsistent (L %d G %d tps %d rows %d)", who, m.L, m.G, m.tps, m.tile_rows);
  OSB_REQUIRE(m.mode == 0 || (m.S > 0 && m.T == m.L), "%s: temporal map needs S > 0 and T == L", who);
  dst->mode = m.mode; dst->L = m.L; dst->S = m.S; dst->T = m.T; dst->G = m.G; dst->tps = m.tps; dst->TR = m.tile_rows;
  return OSB_OK;
}

int make_tile_sets(TileSets* dst, const osb_attn_tiles_args* a, const char* who) {
  OSB_REQUIRE(a->out || a->out_scatter, "%s: null tensor", who);
  const int rc = make_tile_map(&dst->qmap, a->q_map, who);
  if (rc) return rc;
  const int G = a->q_map.G;
  OSB_REQUIRE(a->kv_tile_rows >= 16 && a->kv_tile_rows <= 128 && a->kv_tile_rows % 16 == 0,
              "%s: key tiles must have 16..128 rows in multiples of 16, got %d", who, a->kv_tile_rows);
  OSB_REQUIRE(a->Lk > 0 && a->kv_tiles_per_set >= 1 && (int64_t)a->kv_tiles_per_set * a->kv_tile_rows >= (int64_t)(G > 1 ? G : 1) * a->Lk,
              "%s: %d key tiles of %d rows cannot hold %d keys", who, a->kv_tiles_per_set, a->kv_tile_rows, a->Lk);
  OSB_REQUIRE(G == 1 || (a->kv_tiles_per_set == 1), "%s: packed sequences use one key tile per set", who);
  OSB_REQUIRE(a->num_seqs > 0 && a->num_heads > 0, "%s: empty problem", who);
  OSB_REQUIRE(a->out_ld % 8 == 0 && (reinterpret_cast<uintptr_t>(a->out) & 15) == 0, "%s: out must be 16-byte aligned", who);
  dst->BK = a->kv_tile_rows; dst->nkb = a->kv_tiles_per_set; dst->Lk = a->Lk;
  dst->num_seqs = a->num_seqs;
  dst->num_sets = G > 1 ? (a->num_seqs + G - 1) / G : a->num_seqs;
  dst->kv_lens = a->kv_lens;
  dst->out = static_cast<__nv_bfloat16*>(a->out);
  dst->out_ld = a->out_ld;
  return make_row_scatter(&dst->out_sc, a->out_scatter, a->num_seqs * a->q_map.L, who);
}

int check_attn_short_args(const osb_attn_short_args* a, const char* who) {
  OSB_REQUIRE(a != nullptr, "%s: null args", who);
  OSB_REQUIRE(a->q && a->k && a->v && a->out, "%s: null tensor", who);
  OSB_REQUIRE(a->Lq > 0 && a->Lk > 0 && a->num_seqs > 0 && a->num_heads > 0, "%s: empty problem", who);
  OSB_REQUIRE(a->seqs_per_batch > 0, "%s: seqs_per_batch must be positive", who);
  OSB_REQUIRE((a->q_ld % 8) == 0 && (a->k_ld % 8) == 0 && (a->v_ld % 8) == 0 && (a->out_ld % 8) == 0,
              "%s: leading dimensions must be multiples of 8 elements", who);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(a->q) | reinterpret_cast<uintptr_t>(a->k) |
                reinterpret_cast<uintptr_t>(a->v) | reinterpret_cast<uintptr_t>(a->out)) & 15) == 0,
              "%s: tensors must be 16-byte aligned", who);
  OSB_REQUIRE((a->q_norm_w == nullptr) == (a->k_norm_w == nullptr), "%s: q/k norm weights must come together", who);
  OSB_REQUIRE((a->rope_cos == nullptr) == (a->rope_sin == nullptr), "%s: rope cos/sin must come together", who);
  OSB_REQUIRE((a->q_norm_w2 == nullptr) == (a->k_norm_w2 == nullptr) && (a->q_norm_w2 == nullptr || a->q_norm_w != nullptr),
              "%s: the second norm weight pair needs the first", who);
  OSB_REQUIRE(a->rope_cos == nullptr || ((reinterpret_cast<uintptr_t>(a->rope_cos) | reinterpret_cast<uintptr_t>(a->rope_sin)) & 15) == 0,
              "%s: rope tables must be 16-byte aligned", who);
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
  OSB_REQUIRE(a->q_tiles && a->k_tiles && a->v_tiles, "osb_attn_tiles: null tensor");
  const int D = a->head_dim;
  OSB_REQUIRE(D == 64 || D == 72 || D == 128, "osb_attn_tiles: head_dim %d not built (64, 72, 128)", D);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(a->q_tiles) | reinterpret_cast<uintptr_t>(a->k_tiles) | reinterpret_cast<uintptr_t>(a->v_tiles)) & 15) == 0 &&
              a->q_head_stride % 16 == 0 && a->kv_head_stride % 16 == 0, "osb_attn_tiles: tile buffers must be 16-byte aligned");

  TileAttnParams p = {};
  const int rc = make_tile_sets(&p.ts, a, "osb_attn_tiles");
  if (rc) return rc;
  p.q = static_cast<const uint8_t*>(a->q_tiles);
  p.k = static_cast<const uint8_t*>(a->k_tiles);
  p.v = static_cast<const uint8_t*>(a->v_tiles);
  p.q_head_stride = a->q_head_stride; p.kv_head_stride = a->kv_head_stride;
  p.scale_log2 = a->softmax_scale * 1.4426950408889634f;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (D == 64) return attn_tiles_launch<64>(p, a->num_heads, s);
  if (D == 72) return attn_tiles_launch<72>(p, a->num_heads, s);
  return attn_tiles_launch<128>(p, a->num_heads, s);
}

// Argument checks and launch shared by osb_attn_short and osb_attn_short_bias (bias == nullptr: the plain kernel).
static int attn_short_entry(const osb_attn_short_args* a, const float* bias, int64_t bias_head_stride, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  const int rc = check_attn_short_args(a, "osb_attn_short");
  if (rc) return rc;
  const int D = a->head_dim;
  OSB_REQUIRE(D == 64 || D == 72 || D == 128, "osb_attn_short: head_dim %d not built (64, 72, 128)", D);

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
