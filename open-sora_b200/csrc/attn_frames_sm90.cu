// Frame-causal attention of ONE 512-wide head on sm_90a (osb_attn_frames): out = softmax(q k^T * scale + frame mask) v,
// query token i sees key j iff j < min(Lk, (q_frame0 + i / frame_tokens + 1) * frame_tokens).  Exact online softmax in
// the arithmetic of the other bf16 attention kernels (attn_sm90.cu): fp32 scores in log2 units, guarded running
// maximum, P rounded to bf16 unnormalised, O accumulated and rescaled in fp32, one rounding at the output.
//
// A 64-row x 512-channel fp32 O is half of an SM's register file, so one CTA owns 64 query rows and its two consumer
// warpgroups split the CHANNELS of O (256 each, 128 accumulator registers per thread) and, for S = Q K^T whose
// contraction runs over all 512 channels, the KEYS of a 128-key block (64 each):
//   warpgroup w:  S_w[64 x 64] = Q[64 x 512] K[keys 64 w .. + 63]^T          (32 wgmma m64n64k16, both operands smem)
//                 row maxima of S_w -> shared memory, named barrier, running maximum over both halves (identical in both)
//                 P_w = exp2(S_w * sc - max) -> bf16 -> chunk w of the 128-byte-swizzled P tile, partial row sum l_w
//                 named barrier
//                 O_w[64 x 256] += P[64 x 128] V[128 keys, channels 256 w .. + 255]   (32 wgmma m64n64k16, P the
//                 shared-memory A operand, V the MN-major B operand exactly as it was loaded)
// and the two partial row sums are added once at the end.  Q (64 KB) stays resident; K and V stream as [128 keys x 64
// channels] sub-tiles of 16 KB (one 128-byte swizzle row per key) through ONE ring of 8 stages, 16 sub-tiles per key
// block: K channels 0..7 (both warpgroups read their 64 key rows of each), then V channel groups 0, 4, 1, 5, 2, 6, 3, 7
// (the warpgroups' groups alternate so both can start their PV product at once).  Every consumer waits on every full
// barrier and arrives on every empty barrier, also for the V sub-tiles it does not read, so each barrier sees the same
// two-consumer protocol in every phase.  The loads are 3-D TMA tiles (column, row, sample: rows past Lq / Lk arrive as
// zeros, never as the next sample's rows).
//
// There is no producer warpgroup.  The other warp-specialised kernels spend a warpgroup on the producer and hand its
// registers to the consumers with setmaxnreg; for this kernel ptxas 12.9 kept the consumers of that 384-thread layout
// at 168 registers (32 accumulators in local memory, every wgmma serialised: C7512), and it wants about 200.  So the CTA is
// the two consumer warpgroups alone (256 threads, up to 255 registers) and thread 0 refills the ring in passing:
// whenever its warpgroup releases a sub-tile it waits for the other warpgroup's release of the same stage and issues the
// load of the sub-tile 8 places ahead.  That wait cannot deadlock: the other warpgroup reaches every release of a block
// without needing anything from thread 0 that thread 0 has not already done (the sub-tile's load, the named barriers
// before it).
//
// Key blocks wholly past the tile's last visible key are neither loaded nor computed; the rest are masked per row, so
// a tile may straddle frames.  Work grows with the tile's position: the grid index counts query tiles downwards and the
// heaviest tiles start first.  Keys are never split across CTAs and nothing is accumulated with atomics, so a call
// is deterministic.  Not built: a 2-CTA cluster with multicast of the K / V sub-tiles (DESIGN.md 4.12).
//
// Replaces, in the reference's causal VAE (opensora/models/hunyuan_vae/unet_causal_3d_blocks.py): the dense -inf / 0
// mask of prepare_causal_attention_mask (:52-60), the one-head diffusers Attention built at :311-325 and its call at
// :349-352 (scaled_dot_product_attention over [T h w, T h w] with that mask).
#include "common.cuh"
#include "tiles.cuh"
#include "wgmma.cuh"

namespace osb {

constexpr int kFrD = 512;               // the one head size built
constexpr int kFrRows = 64;             // query rows per CTA
constexpr int kFrKeys = 128;            // keys per online-softmax step
constexpr int kFrStages = 8;            // ring stages = sub-tiles of one operand of a key block
constexpr int kFrThreads = 256;         // two consumer warpgroups; thread 0 also issues the loads
constexpr int kFrQChunk = kFrRows * 128;        // [64 rows x 64 channels] bf16, 128-byte swizzle
constexpr int kFrSub = kFrKeys * 128;           // [128 keys x 64 channels]
constexpr int kFrQBytes = (kFrD / 64) * kFrQChunk;
constexpr int kFrPBytes = 2 * kFrQChunk;        // P[64 x 128]: two [64 rows x 64 keys] chunks, one per warpgroup
constexpr int kFrData = kFrQBytes + kFrPBytes + kFrStages * kFrSub;
constexpr int kFrSmem = 1024 + kFrData + 2 * kFrRows * 4 + 8 * (1 + 2 * kFrStages);   // + alignment slack, row exchange, mbarriers
static_assert(kFrSmem <= 227 * 1024, "shared memory budget of one SM");

struct FrameAttnParams {
  __nv_bfloat16* out;
  int64_t out_ld, q_batch_stride;
  int32_t Lq, Lk, batch, nqt;
  int32_t frame_tokens, q_frame0;
  float scale_log2;
};

__global__ void __launch_bounds__(kFrThreads, 1)
attn_frames_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk,
                   const __grid_constant__ CUtensorMap tv, const FrameAttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 1024-byte aligned
  const uint32_t sQ = base, sP = base + kFrQBytes, sRing = sP + kFrPBytes;
  float* xch = reinterpret_cast<float*>(smem_raw + (base - smem_u32(smem_raw)) + kFrData);   // [2 warpgroups][64 rows]
  const uint32_t bar = base + kFrData + 2 * kFrRows * 4;
  const uint32_t q_full = bar;
  auto full_bar = [&](int s) { return bar + 8u + 8u * s; };
  auto empty_bar = [&](int s) { return bar + 8u + 8u * (kFrStages + s); };
  auto stage = [&](int s) { return sRing + (uint32_t)(s * kFrSub); };

  const int w = threadIdx.x >> 7, tid_wg = threadIdx.x & 127;   // w: warpgroup 0 / 1
  // heaviest tiles first: block 0 takes the last query tile
  const int qt = p.nqt - 1 - (int)(blockIdx.x / (unsigned)p.batch), b = (int)(blockIdx.x % (unsigned)p.batch);
  const int row0 = qt * kFrRows;
  const int hw = p.frame_tokens;
  // keys row i may see: [0, row_limit(i)); rows past Lq compute on zeros with the last row's limit and are not stored
  auto row_limit = [&](int i) {
    i = i < p.Lq ? i : p.Lq - 1;
    const int64_t lim = ((int64_t)p.q_frame0 + i / hw + 1) * hw;
    return (int)(lim < p.Lk ? lim : p.Lk);
  };
  const int nkb = (row_limit(row0 + kFrRows - 1) + kFrKeys - 1) / kFrKeys;   // >= 1

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tq); tma_prefetch_desc(&tk); tma_prefetch_desc(&tv);
    mbar_init(q_full, 1);
    for (int s = 0; s < kFrStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }   // 2: one per consumer
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // q, k, v were written by the previous kernels, which may also still read `out`

  // ring refills by thread 0.  Sub-tile u = 16 kb + (0..7: K channels, 8..15: V groups) lives in stage u % 8; the release
  // of K channel c of block kb is followed by the load of V position c of the same block, the release of V position c by
  // the load of K channel c of the next block.
  const bool loader = threadIdx.x == 0;
  auto load_k = [&](int kb, int c) {
    mbar_expect_tx(full_bar(c), (uint32_t)kFrSub);
    tma_load_3d(&tk, full_bar(c), stage(c), c * 64, kb * kFrKeys, b);
  };
  auto load_v = [&](int kb, int s) {
    mbar_expect_tx(full_bar(s), (uint32_t)kFrSub);
    tma_load_3d(&tv, full_bar(s), stage(s), ((s & 1) * 4 + (s >> 1)) * 64, kb * kFrKeys, b);
  };
  if (loader) {
    mbar_expect_tx(q_full, (uint32_t)kFrQBytes);
    for (int c = 0; c < kFrD / 64; ++c) tma_load_3d(&tq, q_full, sQ + (uint32_t)(c * kFrQChunk), c * 64, row0, b);
    for (int c = 0; c < 8; ++c) load_k(0, c);
  }

  const int lane = tid_wg & 31, quad = lane & 3;
  const int r_loc = (tid_wg >> 5) * 16 + (lane >> 2);   // rows r_loc and r_loc + 8 of the query tile
  const float sc = p.scale_log2;
  const int lim[2] = {row_limit(row0 + r_loc), row_limit(row0 + r_loc + 8)};
  // accumulator fragments: x[4 j + 2 hh + e] = (row r_loc + 8 hh, column 8 j + 2 quad + e); column = key 64 w + .. of the
  // block for s, channel 256 w + 64 i + .. for o[i]
  float s[32], o[4][32];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int x = 0; x < 32; ++x) o[i][x] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t p_mine = sP + (uint32_t)(w * kFrQChunk) + 4u * quad;   // my bf16 pair inside a 16-byte unit of chunk w

  mbar_wait_notrace(q_full, 0u);
  for (int kb = 0; kb < nkb; ++kb) {
    // ---- S_w = Q K_w^T: one K sub-tile (64 channels, 4 k16 steps) at a time, each released when its product retired ----
#pragma unroll
    for (int x = 0; x < 32; ++x) s[x] = 0.f;
    wgmma_fence_regs(s);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      mbar_wait_notrace(full_bar(c), 0u);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        Wgmma<64>::mma(s, make_sw128_kmajor_desc(sQ + (uint32_t)(c * kFrQChunk) + 32u * k),
                       make_sw128_kmajor_desc(stage(c) + (uint32_t)(w * 64 * 128) + 32u * k), 1u);
      wgmma_commit();
      if (c > 0) {
        wgmma_wait<1>();
        if (tid_wg == 0) mbar_arrive(empty_bar(c - 1));
        if (loader) { mbar_wait_notrace(empty_bar(c - 1), 0u); load_v(kb, c - 1); }
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    if (tid_wg == 0) mbar_arrive(empty_bar(7));
    if (loader) { mbar_wait_notrace(empty_bar(7), 0u); load_v(kb, 7); }

    // ---- mask, maximum over this warpgroup's 64 keys, exchange with the other warpgroup ----
    const int key0 = kb * kFrKeys + w * 64 + 2 * quad;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int x = 0; x < 32; ++x) {
      const int hh = (x >> 1) & 1;
      if (key0 + 8 * (x >> 2) + (x & 1) >= lim[hh]) s[x] = -INFINITY;
      mx[hh] = fmaxf(mx[hh], s[x]);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      if (quad == 0) xch[w * kFrRows + r_loc + 8 * hh] = mx[hh];
    }
    // after this barrier both warpgroups have also retired the previous block's PV product: P may be overwritten
    named_barrier_sync(1, 256);
    float alpha[2], ms[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float mn = fmaxf(m[hh], fmaxf(mx[hh], xch[(w ^ 1) * kFrRows + r_loc + 8 * hh]));
      alpha[hh] = (mn == -INFINITY) ? 1.f : fast_exp2((m[hh] - mn) * sc);   // m == -inf: exp2(-inf) = 0
      ms[hh] = (mn == -INFINITY) ? 0.f : mn * sc;
      m[hh] = mn;
      l[hh] *= alpha[hh];
    }
    // ---- P_w = exp2(S_w * sc - max) (masked scores are -inf and give 0) -> bf16 -> chunk w of the P tile ----
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const float p0 = fast_exp2(fmaf(s[4 * j + 2 * hh], sc, -ms[hh]));
        const float p1 = fast_exp2(fmaf(s[4 * j + 2 * hh + 1], sc, -ms[hh]));
        l[hh] += p0 + p1;
        const uint32_t addr = p_mine + sw128_off(r_loc + 8 * hh, j);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_bf16x2(p0, p1)) : "memory");
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int x = 0; x < 32; ++x) o[i][x] *= alpha[(x >> 1) & 1];
    fence_proxy_async_smem();   // P is read by the tensor core through the async proxy
    named_barrier_sync(2, 256);

    const bool more = kb + 1 < nkb;
    // ---- O_w += P V_w: my channel group i sits in stage 2 i + w; 16 keys per k step = two 8-row swizzle atoms ----
#pragma unroll
    for (int i = 0; i < 4; ++i) wgmma_fence_regs(o[i]);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int st = 2 * i + w;
      mbar_wait_notrace(full_bar(st), 1u);
      wgmma_fence();
#pragma unroll
      for (int g = 0; g < 8; ++g)
        WgmmaBT<64>::mma(o[i], make_sw128_kmajor_desc(sP + (uint32_t)((g >> 2) * kFrQChunk) + 32u * (g & 3)),
                         make_sw128_kmajor_desc(stage(st) + 2048u * g), 1u);
      wgmma_commit();
      if (i > 0) {
        wgmma_wait<1>();
        if (tid_wg == 0) mbar_arrive(empty_bar(st - 2));
        if (loader && more) { mbar_wait_notrace(empty_bar(st - 2), 1u); load_k(kb + 1, st - 2); }
      }
    }
    // the other warpgroup's V sub-tiles: waited for and released unread, which keeps this consumer in step with the ring
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int st = 2 * i + (w ^ 1);
      mbar_wait_notrace(full_bar(st), 1u);
      if (tid_wg == 0) mbar_arrive(empty_bar(st));
      if (loader && more) { mbar_wait_notrace(empty_bar(st), 1u); load_k(kb + 1, st); }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 4; ++i) wgmma_fence_regs(o[i]);
    if (tid_wg == 0) mbar_arrive(empty_bar(6 + w));
    if (loader && more) { mbar_wait_notrace(empty_bar(6), 1u); load_k(kb + 1, 6); }
  }
  pdl_launch_dependents();   // every load of this CTA is issued

  // ---- row sums of both key halves, normalise, round once to bf16, store ----
  float inv[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
  }
  // (the other warpgroup read the last block's maxima before the barrier in front of the PV product)
#pragma unroll
  for (int hh = 0; hh < 2; ++hh)
    if (quad == 0) xch[w * kFrRows + r_loc + 8 * hh] = l[hh];
  named_barrier_sync(1, 256);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float lt = l[hh] + xch[(w ^ 1) * kFrRows + r_loc + 8 * hh];
    inv[hh] = lt > 0.f ? 1.0f / lt : 0.f;
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = row0 + r_loc + 8 * hh;
    if (row >= p.Lq) continue;
    __nv_bfloat16* dst = p.out + ((int64_t)b * p.q_batch_stride + row) * p.out_ld + w * 256 + 2 * quad;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(dst + 64 * i + 8 * j) =
            pack_bf16x2(o[i][4 * j + 2 * hh] * inv[hh], o[i][4 * j + 2 * hh + 1] * inv[hh]);
  }
}

int attn_frames_init() {
  OSB_CHECK_CUDA(cudaFuncSetAttribute(attn_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFrSmem));
  return OSB_OK;
}

}  // namespace osb

extern "C" int osb_attn_frames(const osb_attn_frames_args* a, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(a != nullptr, "osb_attn_frames: null args");
  OSB_REQUIRE(a->q && a->k && a->v && a->out, "osb_attn_frames: null tensor");
  OSB_REQUIRE(a->head_dim == kFrD, "osb_attn_frames: head_dim %d not built (512)", a->head_dim);
  OSB_REQUIRE(a->q_ld >= kFrD && a->k_ld >= kFrD && a->v_ld >= kFrD && a->out_ld >= kFrD &&
                  a->q_ld % 8 == 0 && a->k_ld % 8 == 0 && a->v_ld % 8 == 0 && a->out_ld % 8 == 0,
              "osb_attn_frames: leading dimensions must be >= 512 and multiples of 8 (q %lld k %lld v %lld out %lld)",
              (long long)a->q_ld, (long long)a->k_ld, (long long)a->v_ld, (long long)a->out_ld);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(a->q) | reinterpret_cast<uintptr_t>(a->k) | reinterpret_cast<uintptr_t>(a->v) |
                reinterpret_cast<uintptr_t>(a->out)) & 15) == 0, "osb_attn_frames: tensors must be 16-byte aligned");
  OSB_REQUIRE(a->frame_tokens >= 1, "osb_attn_frames: frame_tokens must be >= 1, got %d", a->frame_tokens);
  OSB_REQUIRE(a->batch >= 1 && a->Lq >= 1, "osb_attn_frames: empty problem (batch %d, Lq %lld)", a->batch, (long long)a->Lq);
  OSB_REQUIRE(a->q_frame0 >= 0 && a->Lk >= 1,
              "osb_attn_frames: a query would see no key (q_frame0 %d, Lk %lld)", a->q_frame0, (long long)a->Lk);
  OSB_REQUIRE(a->Lq < (1ll << 31) - kFrRows && a->Lk < (1ll << 31) - kFrKeys, "osb_attn_frames: more than 2^31 tokens");
  OSB_REQUIRE(a->batch == 1 || (a->q_batch_stride >= a->Lq && a->k_batch_stride >= a->Lk),
              "osb_attn_frames: batch strides (%lld, %lld rows) shorter than a sample (%lld, %lld rows)",
              (long long)a->q_batch_stride, (long long)a->k_batch_stride, (long long)a->Lq, (long long)a->Lk);
  OSB_REQUIRE(a->softmax_scale > 0.f, "osb_attn_frames: softmax_scale must be positive");
  const int64_t nqt = (a->Lq + kFrRows - 1) / kFrRows;
  OSB_REQUIRE(nqt * a->batch < (1ll << 31), "osb_attn_frames: grid too large");

  // a single sample has no stride between samples: any valid one serves
  const uint64_t qbs = a->batch == 1 ? (uint64_t)a->Lq : (uint64_t)a->q_batch_stride;
  const uint64_t kbs = a->batch == 1 ? (uint64_t)a->Lk : (uint64_t)a->k_batch_stride;
  CUtensorMap tq, tk, tv;
  int rc = make_tmap_3d_bf16(&tq, a->q, (uint64_t)a->Lq, kFrD, (uint64_t)a->q_ld, (uint64_t)a->batch, qbs * a->q_ld, kFrRows, 64);
  if (rc) return rc;
  rc = make_tmap_3d_bf16(&tk, a->k, (uint64_t)a->Lk, kFrD, (uint64_t)a->k_ld, (uint64_t)a->batch, kbs * a->k_ld, kFrKeys, 64);
  if (rc) return rc;
  rc = make_tmap_3d_bf16(&tv, a->v, (uint64_t)a->Lk, kFrD, (uint64_t)a->v_ld, (uint64_t)a->batch, kbs * a->v_ld, kFrKeys, 64);
  if (rc) return rc;

  FrameAttnParams p = {};
  p.out = static_cast<__nv_bfloat16*>(a->out);
  p.out_ld = a->out_ld;
  p.q_batch_stride = (int64_t)qbs;
  p.Lq = (int32_t)a->Lq; p.Lk = (int32_t)a->Lk; p.batch = a->batch; p.nqt = (int32_t)nqt;
  p.frame_tokens = a->frame_tokens; p.q_frame0 = a->q_frame0;
  p.scale_log2 = a->softmax_scale * 1.4426950408889634f;
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)(nqt * a->batch)), dim3(kFrThreads), kFrSmem,
                                         static_cast<cudaStream_t>(stream), attr);
  OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, attn_frames_kernel, tq, tk, tv, p));
  count_launch();
  return OSB_OK;
}
