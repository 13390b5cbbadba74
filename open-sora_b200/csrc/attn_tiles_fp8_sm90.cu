// FP8 (e4m3) attention over head tiles on sm_90a: the opt-in attention path of STDiT3 (include/osb200.h,
// osb_head_tiles_fp8 / osb_attn_tiles_fp8; tile format in tiles.cuh).
//
//   head_tiles_fp8_kernel  one CTA of 128 threads per (tile, head, kind).  q / k: thread r quantizes row r of the bf16
//                          tile (per-row scale) and stores its 128-byte swizzled e4m3 row.  v: the tile is staged in
//                          shared memory, thread c reduces channel c over the tile's rows and stores the channel's
//                          codes in the vt8 key order.
//   attn_tiles_fp8_kernel  one CTA per (query tile, head), 3 warpgroups, the structure of attn_fp8_kernel: warpgroup 0
//                          (24 registers) has one thread that bulk-copies the Q tile once and streams the set's K / V
//                          tiles with their scales through a 4-stage mbarrier ring; warpgroups 1 and 2 own 64 query rows
//                          each: S = Q K^T by wgmma e4m3 (ceil(D / 32) k32 steps), masks and the online softmax in
//                          registers, P8 = e4m3(256 p) packed from the S accumulator into the register A fragment of the
//                          PV wgmma (N = D), the partial promoted as O = alpha O + s_v (.) partial.  The output rows are
//                          addressed as attn_tiles_kernel addresses them (inverse q map, optional peer scatter).
#include "common.cuh"
#include "stage.cuh"
#include "tiles.cuh"
#include "wgmma.cuh"

namespace osb {

constexpr int kTF8Stages = 4;
constexpr int kTF8Threads = 384;
constexpr int kTF8StageBytes = 2 * kTileF8Bytes + 1024;   // K tile, V tile (D <= 128 rows), k scales, v scales
constexpr int kTF8Smem = 1024 + kTileF8Bytes + kTF8Stages * kTF8StageBytes + 8 * (1 + 2 * kTF8Stages);

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
      uint4 o;
      o.x = e4m3x2(x[0] / s, x[1] / s) | (e4m3x2(x[2] / s, x[3] / s) << 16);
      o.y = e4m3x2(x[4] / s, x[5] / s) | (e4m3x2(x[6] / s, x[7] / s) << 16);
      o.z = e4m3x2(x[8] / s, x[9] / s) | (e4m3x2(x[10] / s, x[11] / s) << 16);
      o.w = e4m3x2(x[12] / s, x[13] / s) | (e4m3x2(x[14] / s, x[15] / s) << 16);
      *reinterpret_cast<uint4*>(dst + r * 128 + ((w ^ (r & 7)) << 4)) = o;
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
      for (int w = 0; w < 8; ++w) {   // key positions 16 w .. 16 w + 15
        uint32_t q[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int pos = 16 * w + 4 * k;
          const float x0 = __bfloat162float(tile[vt8_key(pos)][c]), x1 = __bfloat162float(tile[vt8_key(pos + 1)][c]);
          const float x2 = __bfloat162float(tile[vt8_key(pos + 2)][c]), x3 = __bfloat162float(tile[vt8_key(pos + 3)][c]);
          q[k] = e4m3x2(x0 / s, x1 / s) | (e4m3x2(x2 / s, x3 / s) << 16);
        }
        *reinterpret_cast<uint4*>(dst + c * 128 + ((w ^ (c & 7)) << 4)) = make_uint4(q[0], q[1], q[2], q[3]);
      }
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
  TileMap qmap;
  int32_t BK, nkb, Lk;
  int64_t num_seqs;
  const int32_t* kv_lens;
  __nv_bfloat16* out;
  int64_t out_ld;
  float sc;   // softmax_scale * log2(e)
  RowScatter out_sc;
};

// valid key slots of a set: packed tiles G * Lk, else Lk clipped by kv_lens
__device__ __forceinline__ int tile_set_keys(const TileFp8Attn& p, int64_t set) {
  int keys = p.qmap.G > 1 ? p.qmap.G * p.Lk : p.Lk;
  if (p.qmap.G == 1 && p.kv_lens) { const int l = __ldg(p.kv_lens + set); keys = l < keys ? (l < 0 ? 0 : l) : keys; }
  return keys;
}

template <int D>
__global__ void __launch_bounds__(kTF8Threads, 1) attn_tiles_fp8_kernel(const TileFp8Attn p) {
  constexpr int KSTEPS = (D + 31) / 32;   // k32 steps of QK^T: the codes past D are zero
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

  const int wg = threadIdx.x >> 7, tid_wg = threadIdx.x & 127;
  const int64_t qtile = blockIdx.x;
  const int head = blockIdx.y;
  const int64_t set = qtile / p.qmap.tps;
  const int qt = (int)(qtile - set * p.qmap.tps);
  const int keys = tile_set_keys(p, set);
  const int nkt = (keys + p.BK - 1) / p.BK;   // key tiles holding valid keys
  const int64_t qti = (int64_t)head * p.q_head_tiles + qtile;
  const int64_t kti0 = (int64_t)head * p.kv_head_tiles + set * p.nkb;

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
    lo[hh] = hi[hh] = 0;
    if (p.qmap.G > 1) {
      const int g = r / p.qmap.L;
      pos[hh] = r - g * p.qmap.L;
      seq[hh] = set * p.qmap.G + g;
      valid[hh] = g < p.qmap.G && seq[hh] < p.num_seqs;
      if (valid[hh]) { lo[hh] = g * p.Lk; hi[hh] = lo[hh] + p.Lk; }
    } else {
      pos[hh] = qt * p.qmap.TR + r;
      seq[hh] = set;
      valid[hh] = r < p.qmap.TR && pos[hh] < p.qmap.L;
      if (valid[hh]) hi[hh] = keys;
    }
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
    // ---- S = Q K^T ----
    const uint64_t dk = make_sw128_kmajor_desc(sK(stage));
    wgmma_fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k) WgmmaFp8<128>::mma(s, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    // ---- scores in log2 units, masks, running maximum ----
    const float* skp = sk_gen + (kTF8StageBytes / 4) * stage;
    const int slot0 = kb * p.BK;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float2 sk = *reinterpret_cast<const float2*>(skp + 8 * j + 2 * quad);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * j + 2 * quad + e, slot = slot0 + col;
          float v = s[4 * j + 2 * hh + e] * sq[hh] * (e ? sk.y : sk.x);
          if (col >= p.BK || slot < lo[hh] || slot >= hi[hh]) v = -INFINITY;
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
    // ---- partial = P8 V8 (tensor core), then O = alpha O + s_v (.) partial in fp32 ----
    // the v scales are read before the product: once the warpgroup's wgmma retired, every warp is done with the stage
    const float* svp = sv_gen + (kTF8StageBytes / 4) * stage;
    float2 sv[D / 8];
#pragma unroll
    for (int j = 0; j < D / 8; ++j) sv[j] = *reinterpret_cast<const float2*>(svp + 8 * j + 2 * quad);
    const uint64_t dv = make_sw128_kmajor_desc(sV(stage));
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
    if (tid_wg == 0) mbar_arrive(empty_bar(stage));
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      o[4 * j] += sv[j].x * part[4 * j]; o[4 * j + 1] += sv[j].y * part[4 * j + 1];
      o[4 * j + 2] += sv[j].x * part[4 * j + 2]; o[4 * j + 3] += sv[j].y * part[4 * j + 3];
    }
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
    int64_t orow = row_of_token(p.qmap, seq[hh], pos[hh]);
    __nv_bfloat16* obase = p.out;
    if (p.out_sc.mode != 0) {
      int peer;
      scatter_row(p.out_sc, orow, peer, orow);
      obase = static_cast<__nv_bfloat16*>(scatter_base(p.out_sc, peer));
    }
    __nv_bfloat16* dst = obase + orow * p.out_ld + (int64_t)head * D;
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j + 2 * quad) = pack_bf16x2(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
  }
}

int attn_tiles_fp8_init() {
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_fp8_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTF8Smem));
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_tiles_fp8_kernel<72>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTF8Smem));
  return OSB_OK;
}

}  // namespace osb

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
  OSB_REQUIRE(ops->q8 && ops->k8 && ops->v8 && ops->s_q && ops->s_k && ops->s_v && (a->out || a->out_scatter),
              "osb_attn_tiles_fp8: null tensor");
  const int D = a->head_dim;
  OSB_REQUIRE(D == 64 || D == 72, "osb_attn_tiles_fp8: head_dim %d not built (64, 72)", D);
  const osb_tile_map& m = a->q_map;
  OSB_REQUIRE(m.mode == 0 || m.mode == 1, "osb_attn_tiles_fp8: unknown tile map mode %d", m.mode);
  OSB_REQUIRE(m.L > 0 && m.G >= 1 && m.tile_rows > 0 && m.tile_rows <= 128 && m.tile_rows % 8 == 0,
              "osb_attn_tiles_fp8: bad q tile map (L %d G %d rows %d)", m.L, m.G, m.tile_rows);
  OSB_REQUIRE(m.G == 1 ? (m.tps == (m.L + m.tile_rows - 1) / m.tile_rows) : (m.G * m.L <= m.tile_rows && m.tps == 1),
              "osb_attn_tiles_fp8: q tile map inconsistent (L %d G %d tps %d rows %d)", m.L, m.G, m.tps, m.tile_rows);
  OSB_REQUIRE(m.mode == 0 || (m.S > 0 && m.T == m.L), "osb_attn_tiles_fp8: temporal map needs S > 0 and T == L");
  OSB_REQUIRE(a->kv_tile_rows >= 16 && a->kv_tile_rows <= 128 && a->kv_tile_rows % 16 == 0,
              "osb_attn_tiles_fp8: key tiles must have 16..128 rows in multiples of 16, got %d", a->kv_tile_rows);
  OSB_REQUIRE(a->Lk > 0 && a->kv_tiles_per_set >= 1 && (int64_t)a->kv_tiles_per_set * a->kv_tile_rows >= (int64_t)(m.G > 1 ? m.G : 1) * a->Lk,
              "osb_attn_tiles_fp8: %d key tiles of %d rows cannot hold %d keys", a->kv_tiles_per_set, a->kv_tile_rows, a->Lk);
  OSB_REQUIRE(m.G == 1 || (a->kv_tiles_per_set == 1), "osb_attn_tiles_fp8: packed sequences use one key tile per set");
  OSB_REQUIRE(a->num_seqs > 0 && a->num_heads > 0 && a->num_heads <= 65535, "osb_attn_tiles_fp8: empty problem");
  OSB_REQUIRE(a->out_ld % 8 == 0 && (reinterpret_cast<uintptr_t>(a->out) & 15) == 0, "osb_attn_tiles_fp8: out must be 16-byte aligned");
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(ops->q8) | reinterpret_cast<uintptr_t>(ops->k8) | reinterpret_cast<uintptr_t>(ops->v8) |
                reinterpret_cast<uintptr_t>(ops->s_q) | reinterpret_cast<uintptr_t>(ops->s_k) |
                reinterpret_cast<uintptr_t>(ops->s_v)) & 15) == 0,
              "osb_attn_tiles_fp8: e4m3 tiles and scales must be 16-byte aligned");
  const int64_t num_sets = m.G > 1 ? (a->num_seqs + m.G - 1) / m.G : a->num_seqs;
  const int64_t qtiles = num_sets * m.tps;
  OSB_REQUIRE(ops->q_head_tiles >= qtiles && ops->kv_head_tiles >= num_sets * a->kv_tiles_per_set,
              "osb_attn_tiles_fp8: %lld / %lld tiles per head hold less than %lld query / %lld key tiles",
              (long long)ops->q_head_tiles, (long long)ops->kv_head_tiles, (long long)qtiles,
              (long long)(num_sets * a->kv_tiles_per_set));
  OSB_REQUIRE(qtiles < (1ll << 31), "osb_attn_tiles_fp8: problem too large (%lld query tiles)", (long long)qtiles);

  TileFp8Attn p = {};
  p.q8 = static_cast<const uint8_t*>(ops->q8);
  p.k8 = static_cast<const uint8_t*>(ops->k8);
  p.v8 = static_cast<const uint8_t*>(ops->v8);
  p.s_q = ops->s_q; p.s_k = ops->s_k; p.s_v = ops->s_v;
  p.q_head_tiles = ops->q_head_tiles; p.kv_head_tiles = ops->kv_head_tiles;
  p.qmap.mode = m.mode; p.qmap.L = m.L; p.qmap.S = m.S; p.qmap.T = m.T; p.qmap.G = m.G; p.qmap.tps = m.tps; p.qmap.TR = m.tile_rows;
  p.BK = a->kv_tile_rows; p.nkb = a->kv_tiles_per_set; p.Lk = a->Lk;
  p.num_seqs = a->num_seqs;
  p.kv_lens = a->kv_lens;
  p.out = static_cast<__nv_bfloat16*>(a->out);
  p.out_ld = a->out_ld;
  p.sc = a->softmax_scale * 1.4426950408889634f;
  {
    const int rc = make_row_scatter(&p.out_sc, a->out_scatter, a->num_seqs * m.L, "osb_attn_tiles_fp8");
    if (rc) return rc;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)qtiles, (unsigned)a->num_heads), dim3(kTF8Threads), kTF8Smem, s, attr);
  if (D == 64) { OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_tiles_fp8_kernel<64>, p)); }
  else { OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_tiles_fp8_kernel<72>, p)); }
  count_launch();
  return OSB_OK;
}
