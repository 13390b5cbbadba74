// bf16 GEMM for sm_90a:  D[M,N] = epilogue(A[M,K] * W[N,K]^T + bias)
//
// Warp-specialised persistent kernel over 128 x BLOCK_N output tiles: one CTA per SM (at most), CTA b computes tiles
// b, b + gridDim.x, b + 2 gridDim.x, ...  Warpgroup 0 is the producer: one thread streams the A and W tiles with TMA
// into 128-byte-swizzled shared memory (BLOCK_K = 64 bf16 = one swizzle row) through a ring of mbarrier-guarded
// stages.  Warpgroups 1 and 2 each own 64 accumulator rows: wgmma.mma_async reads both operands straight from the
// swizzled tiles (matrix descriptors), the fp32 accumulator lives in registers and the epilogue runs on those
// registers, so the accumulator never goes through memory before its single rounding to bf16.
// One wgmma group stays in flight while the next stage is waited for; a stage is handed back to the producer as soon
// as the group that read it has retired.  The ring's stage and phase run on across tiles, so the producer fills the
// ring with the next tile's k-blocks while the consumers are still in the current tile's epilogue.
// Every mode whose output is a bf16 [rows, N] tile (all but kHeadTiles, kText and the FP8-emitting GELU) stages its
// epilogue through shared memory: the producer TMA-loads the residual tile into an epilogue buffer during the main loop,
// the consumers round each result once into that buffer, over the residual, and one thread writes the tile with TMA
// stores clipped to the output's extents.  No global load then waits behind a global store.  The buffer is reused by
// every tile of the CTA: once the stores have read it, the store thread arrives on `epi_free`, and only then does the
// next tile's residual (or, without a residual, the next tile's results) go into it.
//
// The same main loop serves five front ends (template kMode):
//   kPlain      nn.Linear with fused bias / GELU(tanh) / gate * x + residual epilogues;
//   kConv       causal 3D convolution as implicit GEMM: every k-block is ONE 5-D TMA box of the padded NDHWC input;
//   kHeadTiles  q / k / v projection whose epilogue writes per-head operand tiles (tiles.cuh) with RMSNorm + RoPE;
//   kLora       kPlain plus an unmerged low-rank update: after the K loop the producer streams ceil(r / 64) more
//               k-blocks, U = x A^T [M, r] in the A slot and s B [N, r] in the W slot, through the same stage ring, so
//               A W^T + U (s B)^T lands in one fp32 accumulator before the unchanged epilogue; with a DoRA column
//               scale the accumulator is multiplied by col_scale[n] in registers first.
//   kText       nn.Linear with the text encoders' activations: T5's gated GELU gelu_tanh(x wi_0^T) * (x wi_1^T) over a
//               weight whose rows interleave wi_0 and wi_1 (both halves of an output column sit in one thread's
//               accumulator pair, the [M, 2 d_ff] product never leaves registers), and CLIP's bias + quick GELU.
//   kFp8        kPlain on e4m3 operands with per-row scales: a k-block is 128 e4m3 elements (the same 128-byte swizzle row,
//               box bytes and stage ring as 64 bf16), issued as 4 wgmma k32 steps into a partial accumulator that is added
//               into the fp32 register accumulator after every k-block; the epilogue scales the accumulator by
//               a_scale[row] * w_scale[col] before the unchanged bias / GELU / gate + residual code.  BLOCK_N 64 / 128.
//   kFp8Blk     kFp8 with 1 x 128 block scales on A: each k-block's partial is multiplied by a_scale[row, kb] as it is
//               promoted into the fp32 accumulator (per-row scales are a zero k-stride), the epilogue applies w_scale[col].
//               With BLOCK_N = 128 it also has the FP8-emitting GELU epilogue: one output tile row is exactly one
//               128-column scale block, held by the 4 lanes of a quad, so the block amax is two shuffles; the codes and
//               the scale go out instead of bf16.
//   kFp8BlkLora kFp8Blk plus an unmerged low-rank update, as kLora adds one to kPlain: after the e4m3 k-blocks the
//               producer streams ceil(r / 64) bf16 k-blocks of U = x A^T [M, r] and s B [N, r] through the same ring (64
//               bf16 and 128 e4m3 elements are both one 128-byte swizzle row).  Before the first of them the accumulator
//               is multiplied by w_scale[col], which scales the FP8 sum only; each bf16 k-block is summed into the partial
//               accumulator by 4 wgmma k16 steps and promoted unscaled, then the optional DoRA column scale multiplies
//               the total before the unchanged epilogue (the FP8-emitting GELU included).
//
// Replaces every nn.Linear on the denoiser block path of the reference
// (opensora/models/mmdit/layers.py:209-214,247-252,277-281,314-334,401) and the fused epilogues
// replace the separate bias / GELU(tanh) / gate*x+residual elementwise kernels.
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"
#include "tiles.cuh"
#include "wgmma.cuh"

namespace osb {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kNumThreads = 384;            // producer warpgroup + two consumer warpgroups
constexpr int kStageBudget = 200 * 1024;    // operand ring of the register-epilogue modes (one CTA per SM)
constexpr int kSmemLimit = 227 * 1024;      // sm_90 per-block dynamic shared memory limit

enum { kPlain = 0, kConv = 1, kHeadTiles = 2, kLora = 3, kText = 4, kFp8 = 5, kFp8Blk = 6, kFp8BlkLora = 7 };

// kFp8Blk / kFp8BlkLora only: where the scale of (row m, k-block kb) of A is (a_scale + m * a_ld + kb * a_kstride;
// a_kstride = 0 for per-row scales), the e4m3 output of the FP8-emitting GELU epilogue (codes d8 [M, N], ldd8; scales
// [M, N / 128]) and, kFp8BlkLora only, the optional DoRA column scale (null: none).
struct Fp8BlockParams {
  int64_t a_ld, a_kstride;
  uint8_t* d8;
  float* d_scale;
  int64_t ldd8, ld_dscale;
  const float* col_scale;
};

struct GemmEpilogueParams {
  const __nv_bfloat16* bias;
  __nv_bfloat16* D;
  const __nv_bfloat16* R;
  const float* gate;
  const int32_t* mod_index;
  int64_t M, N, K;
  int64_t ldd, ldr;
  int64_t group_rows;
  int64_t gate_stride;
  int32_t epilogue;
};

// Head-tile epilogue (kHeadTiles): every output row is split into heads of D = BLOCK_N / 2 columns; per head: bias,
// optional RMSNorm (fp32 statistics over the fp32 accumulator), optional interleaved-pair RoPE by token position, one
// rounding to bf16, stored at the row's place inside the head's operand tile (tiles.cuh) - the projection output never
// exists in token layout.  Column group kidx = col / C (C = heads * D) selects the kind (q / k / v) = kidx % nkinds.
struct HeadTileParams {
  uint8_t* base;
  int64_t kind_stride, head_stride;
  TileMap map;
  int32_t tile_bytes;
  int32_t heads, nkinds;
  uint32_t norm_mask, rope_mask;
  const __nv_bfloat16* norm_w[4];
  float eps;
  const float* cos;
  const float* sin;
};

// Implicit-GEMM view of a causal 3D convolution over a (replicate-)padded NDHWC activation tensor: one
// output tile is a Tt x Ht x Wt box of output positions (128 rows).  The K loop walks (kt, kh, kw) taps x 64-channel
// chunks; every k-block is ONE 5-D TMA box load at the tap's offset.
struct ConvGeom {
  int32_t wt_log2, ht_log2;              // box: Wt = 1 << wt_log2, Ht = 1 << ht_log2, Tt = 128 / (Wt * Ht)
  int32_t tiles_w, tiles_h, tiles_t, nb; // tiles per dimension, batch
  int32_t w_out, h_out, t_out;
  int32_t sw, sh, st;                    // convolution strides
  int32_t kw_n, kh_n;                    // taps along w, h (taps along t = k-blocks / (kw_n * kh_n * cin_chunks))
  int32_t cin_chunks;                    // 64-wide channel chunks per tap
};

// Modes whose output is a bf16 [rows, N] tile go through the staged epilogue: the 128 x BLOCK_N tile is assembled in a
// shared-memory buffer (the residual tile is TMA-loaded into it during the main loop) and leaves by TMA tile stores.
__host__ __device__ constexpr bool staged_epilogue(int mode) {
  return mode == kPlain || mode == kConv || mode == kLora || mode == kFp8 || mode == kFp8Blk || mode == kFp8BlkLora;
}
__host__ __device__ constexpr bool fp8_mode(int mode) { return mode == kFp8 || mode == kFp8Blk || mode == kFp8BlkLora; }
__host__ __device__ constexpr bool lora_mode(int mode) { return mode == kLora || mode == kFp8BlkLora; }

template <int BLOCK_N, bool kStaged = false>
struct GemmCfg {
  static constexpr int A_BYTES = kBlockM * kBlockK * 2;
  static constexpr int B_BYTES = BLOCK_N * kBlockK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // epilogue buffer: BLOCK_N / 64 boxes of 128 rows x 64 columns (one 128-byte swizzle row per tile row)
  static constexpr int EPI_BYTES = kStaged ? kBlockM * BLOCK_N * 2 : 0;
  static constexpr int RING_BUDGET = kStaged ? kSmemLimit - 1024 - 256 - EPI_BYTES : kStageBudget;
  static constexpr int STAGES_RAW = RING_BUDGET / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;
  static constexpr int NUM_BARS = 2 * STAGES + (kStaged ? 2 : 0);   // full / empty per stage (+ residual, buffer free)
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 1024 + 8 * NUM_BARS;  // +1024 alignment slack
  static_assert(STAGES >= 2, "pipeline needs at least two stages");
  static_assert(SMEM_BYTES <= kSmemLimit, "shared memory");
  static_assert(B_BYTES % 1024 == 0, "W tile must keep 1024-byte swizzle-atom alignment");
  static_assert(BLOCK_N % 16 == 0 && BLOCK_N <= 256, "wgmma N");
  static_assert(!kStaged || BLOCK_N % 64 == 0, "the staged epilogue moves 64-column boxes");
};

template <int BLOCK_N, int kMode>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                 const GemmEpilogueParams p, const ConvGeom cg, const HeadTileParams ht,
                 const __grid_constant__ CUtensorMap tmap_u, const __grid_constant__ CUtensorMap tmap_lb,
                 const int32_t lora_k_blocks,     // kLora / kFp8BlkLora: U / s B maps and ceil(r / 64)
                 const float* a_scale, const float* w_scale,     // kFp8: row scales of A and W; kLora: w_scale is the
                                                                 // optional per-column (DoRA) scale, may be null
                 const Fp8BlockParams fb,                        // kFp8Blk / kFp8BlkLora only
                 const __grid_constant__ CUtensorMap tmap_r,     // staged epilogue: residual (read only when p.R)
                 const __grid_constant__ CUtensorMap tmap_d) {   //   and output, extents exactly those of the output
  constexpr bool kStaged = staged_epilogue(kMode);
  using Cfg = GemmCfg<BLOCK_N, kStaged>;
  constexpr int kStages = Cfg::STAGES;
  constexpr int kBK = fp8_mode(kMode) ? 2 * kBlockK : kBlockK;   // elements per k-block: always 128 bytes per row
  constexpr uint32_t kEpiBoxBytes = kBlockM * 128;   // one 128-row x 64-column box of the epilogue buffer

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 1024-byte aligned
  const uint32_t epi_base = smem_base + kStages * Cfg::STAGE_BYTES;   // staged epilogue buffer (1024-byte aligned)
  const uint32_t bar_base = epi_base + Cfg::EPI_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  const uint32_t res_bar = bar_base + 8u * (2 * kStages);       // staged epilogue: the residual tile has landed
  const uint32_t epi_free = bar_base + 8u * (2 * kStages + 1);  //   the previous tile's stores have read the buffer
  auto smem_a = [&](int s) { return smem_base + s * Cfg::STAGE_BYTES; };
  auto smem_b = [&](int s) { return smem_base + s * Cfg::STAGE_BYTES + Cfg::A_BYTES; };

  const int wg = threadIdx.x >> 7;
  const int tid_wg = threadIdx.x & 127;
  const int64_t num_n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int64_t num_m_blocks =
      kMode == kConv ? (int64_t)cg.nb * cg.tiles_t * cg.tiles_h * cg.tiles_w : (p.M + kBlockM - 1) / kBlockM;
  const int64_t num_tiles = num_m_blocks * num_n_blocks;
  const int64_t num_k_blocks = (p.K + kBK - 1) / kBK;
  const int64_t total_k_blocks = lora_mode(kMode) ? num_k_blocks + lora_k_blocks : num_k_blocks;
  // Tile t -> (m_blk, n_blk), in the order of the grid's CTAs: the tiles in flight at once share A panels and W.  conv:
  // m_blk -> (batch, t-tile, h-tile, w-tile), the box origin in OUTPUT coordinates.
  struct Tile {
    int64_t m_blk, n_blk;
    int n_i, t0, h0, w0;
  };
  auto tile_at = [&](int64_t t) {
    Tile tl = {t / num_n_blocks, t % num_n_blocks, 0, 0, 0, 0};
    if constexpr (kMode == kConv) {
      const int tw = (int)(tl.m_blk % cg.tiles_w);
      const int th = (int)((tl.m_blk / cg.tiles_w) % cg.tiles_h);
      const int tt = (int)((tl.m_blk / ((int64_t)cg.tiles_w * cg.tiles_h)) % cg.tiles_t);
      tl.n_i = (int)(tl.m_blk / ((int64_t)cg.tiles_w * cg.tiles_h * cg.tiles_t));
      tl.w0 = tw << cg.wt_log2;
      tl.h0 = th << cg.ht_log2;
      tl.t0 = tt * (128 >> (cg.wt_log2 + cg.ht_log2));
    }
    return tl;
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_w);
    if constexpr (lora_mode(kMode)) {
      tma_prefetch_desc(&tmap_u);
      tma_prefetch_desc(&tmap_lb);
    }
    if constexpr (kStaged) {
      if (p.R != nullptr) tma_prefetch_desc(&tmap_r);
      tma_prefetch_desc(&tmap_d);
      mbar_init(res_bar, 1);
      mbar_init(epi_free, 1);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel's tail; its outputs are visible from here on

  // The producer needs few registers and the consumers hold up to 128 accumulators each plus the tile loop's state:
  // 128 x 40 + 256 x 232 registers are what the 384 x 168 of one CTA per SM allow.
  if (wg == 0) {
    // ===================== TMA producer (A and W tiles) =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (tid_wg == 0) {
      int stage = 0;
      uint32_t phase = 0;
      uint32_t it = 0;   // this CTA's tile count
      for (int64_t t = blockIdx.x; t < num_tiles; t += gridDim.x, ++it) {
        const Tile tl = tile_at(t);
        const int32_t a_row = (int32_t)(tl.m_blk * kBlockM);
        const int32_t w_row = (int32_t)(tl.n_blk * BLOCK_N);
        auto load_k_block = [&](int64_t kb) {
          mbar_wait_notrace(empty_bar(stage), phase ^ 1);
          mbar_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);   // out-of-bounds box elements are zero filled and counted
          if (lora_mode(kMode) && kb >= num_k_blocks) {   // the rank tail beyond r is zero filled in both U and s B
            const int32_t lk0 = (int32_t)(kb - num_k_blocks) * kBlockK;
            tma_load_2d(&tmap_u, full_bar(stage), smem_a(stage), lk0, a_row);
            tma_load_2d(&tmap_lb, full_bar(stage), smem_b(stage), lk0, w_row);
          } else {
            const int32_t k0 = (int32_t)(kb * kBK);
            if constexpr (kMode == kConv) {   // tap offsets in the padded input, output origin scaled by the stride
              const int tap = (int)(kb / cg.cin_chunks);
              const int32_t ac = (int32_t)(kb - (int64_t)tap * cg.cin_chunks) * kBlockK;
              const int32_t aw = tl.w0 * cg.sw + tap % cg.kw_n;
              const int32_t ah = tl.h0 * cg.sh + (tap / cg.kw_n) % cg.kh_n;
              const int32_t at = tl.t0 * cg.st + tap / (cg.kw_n * cg.kh_n);
              tma_load_5d(&tmap_a, full_bar(stage), smem_a(stage), ac, aw, ah, at, tl.n_i);
            } else {
              tma_load_2d(&tmap_a, full_bar(stage), smem_a(stage), k0, a_row);
            }
            tma_load_2d(&tmap_w, full_bar(stage), smem_b(stage), k0, w_row);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        };
        int64_t kb = 0;
        if constexpr (kStaged) {
          // The residual tile goes into the epilogue buffer, which the previous tile's output stores may still be
          // reading.  So the ring is filled first (those loads need only stages the previous tile has released, and
          // overlap its epilogue), then the buffer is waited for and the residual issued: its latency hides behind the
          // rest of the main loop.  R may alias D (in-place update): each tile has exactly one owner CTA, which reads
          // and writes it.  Boxes past N are not issued; the out-of-bounds part of a box is zero filled and counted.
          if (p.R != nullptr) {
            for (; kb < min((int64_t)kStages, total_k_blocks); ++kb) load_k_block(kb);
            if (it > 0) mbar_wait_notrace(epi_free, (it - 1) & 1u);
            const int live = (int)min((int64_t)(BLOCK_N / 64), (p.N - w_row + 63) / 64);
            mbar_expect_tx(res_bar, (uint32_t)live * kEpiBoxBytes);
            for (int c = 0; c < live; ++c) {
              if constexpr (kMode == kConv)
                tma_load_5d(&tmap_r, res_bar, epi_base + c * kEpiBoxBytes, w_row + 64 * c, tl.w0, tl.h0, tl.t0, tl.n_i);
              else
                tma_load_2d(&tmap_r, res_bar, epi_base + c * kEpiBoxBytes, w_row + 64 * c, a_row);
            }
          }
        }
        for (; kb < total_k_blocks; ++kb) load_k_block(kb);
      }
      pdl_launch_dependents();  // all loads issued: dependents may start filling SMs as they are vacated
    }
    return;
  }

  // ===================== consumers: wgmma main loop =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int cw = wg - 1;   // accumulator rows [64 cw, 64 cw + 64) of the tile
  int stage = 0;
  uint32_t phase = 0;
  uint32_t it = 0;   // this CTA's tile count
  // The previous tile's output stores must have read the epilogue buffer before the buffer takes this tile's residual
  // or results.  The store thread waits for that only once its warpgroup has issued this tile's first k-block, so the
  // wait overlaps the tensor core, and then frees the buffer (epi_free completes phase it - 1).
  auto release_epi_buffer = [&](int64_t kb) {
    if constexpr (kStaged) {
      if (kb == 0 && it > 0 && threadIdx.x == 128) {
        bulk_wait_group_read_all();
        mbar_arrive(epi_free);
      }
    }
  };
  for (int64_t t = blockIdx.x; t < num_tiles; t += gridDim.x, ++it) {
    const Tile tl = tile_at(t);
    const int64_t m_blk = tl.m_blk, n_blk = tl.n_blk;
    // accumulator fragment: acc[4 j + 2 h + e] = (row 16 warp + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e)
    const int warp_in = tid_wg >> 5, lane = tid_wg & 31;
    const int r_frag = cw * 64 + warp_in * 16 + (lane >> 2);
    const int c_frag = 2 * (lane & 3);
    // Staged epilogue: the per-row gate row (modulation group, then mod_index) and FP8 row scale depend on the tile
    // only, so their loads are issued here and their latency hides behind the main loop.  Rows >= M are clamped.
    const float* gate_row[2] = {nullptr, nullptr};
    float sa[2] = {0.f, 0.f};
    if constexpr (kStaged && kMode != kConv) {
      const uint32_t group_rows32 = (uint32_t)(p.group_rows > 0xffffffffll ? 0xffffffffu : p.group_rows);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = min(m_blk * kBlockM + r_frag + 8 * h, p.M - 1);
        if (p.epilogue == OSB_EPI_BIAS_GATE_RES && p.gate != nullptr) {   // modulation group per row: tiles may straddle
          int64_t gi = (uint32_t)row / group_rows32;
          if (p.mod_index) gi = p.mod_index[gi];
          gate_row[h] = p.gate + gi * p.gate_stride;
        }
        if constexpr (kMode == kFp8) sa[h] = __ldg(a_scale + row);
      }
    }
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    if constexpr (fp8_mode(kMode)) {
      // FP8 wgmma adds into its accumulator with fewer mantissa bits than an fp32 add, so a K-long sum in the wgmma
      // accumulator loses precision with K.  Each k-block (128 e4m3 elements) is summed into `part` by the tensor core and
      // promoted into the fp32 register accumulator `acc` before the next one: acc is an fp32 sum of 128-element partials.
      // (Two accumulators per thread: BLOCK_N <= 128 fits the consumers' 232 registers with room to spare.)
      float part[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) part[i] = 0.f;
      // kFp8Blk: the scale rows of this thread's two accumulator rows (clamped: rows >= M are computed but never stored)
      const float* sa_row0 = a_scale;
      const float* sa_row1 = a_scale;
      if constexpr (kMode != kFp8) {
        const int64_t r0 = m_blk * kBlockM + cw * 64 + (tid_wg >> 5) * 16 + ((tid_wg & 31) >> 2);
        sa_row0 = a_scale + min(r0, p.M - 1) * fb.a_ld;
        sa_row1 = a_scale + min(r0 + 8, p.M - 1) * fb.a_ld;
      }
      // One k-block: e4m3 (4 wgmma k32 steps, promoted with its A scales) or, is_tail (kFp8BlkLora's rank tail), bf16
      // (4 wgmma k16 steps, promoted with scale 1: fmaf(p, 1, a) is p + a, one rounding).  Both step 32 bytes along K.
      auto k_block = [&](int64_t kb, auto is_tail) {
        constexpr bool tail = decltype(is_tail)::value;
        float s0 = 1.f, s1 = 1.f;
        if constexpr (kMode != kFp8 && !tail) {   // issued before the wait: the loads overlap the TMA and the tensor core
          s0 = __ldg(sa_row0 + kb * fb.a_kstride);
          s1 = __ldg(sa_row1 + kb * fb.a_kstride);
        }
        if constexpr (tail) {
          // w_scale scales the FP8 sum only: applied once, before the tail's first k-block is promoted (a thread's
          // columns are the same for both of its rows; columns >= N are clamped, never stored)
          if (kb == num_k_blocks) {
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
              const int64_t n = min(n_blk * BLOCK_N + 8 * j + c_frag, p.N - 2);
              const float2 sw = __ldg(reinterpret_cast<const float2*>(w_scale + n));
              acc[4 * j] = __fmul_rn(acc[4 * j], sw.x);
              acc[4 * j + 1] = __fmul_rn(acc[4 * j + 1], sw.y);
              acc[4 * j + 2] = __fmul_rn(acc[4 * j + 2], sw.x);
              acc[4 * j + 3] = __fmul_rn(acc[4 * j + 3], sw.y);
            }
          }
        }
        mbar_wait_notrace(full_bar(stage), phase);
        const uint64_t da = make_sw128_kmajor_desc(smem_a(stage) + (uint32_t)(cw * 64 * 128));
        const uint64_t db = make_sw128_kmajor_desc(smem_b(stage));
        wgmma_fence_regs(part);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // +32 bytes along K per step = +2 in the descriptor's 16-byte units
          if constexpr (tail)
            Wgmma<BLOCK_N>::mma(part, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
          else
            WgmmaFp8<BLOCK_N>::mma(part, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), k > 0 ? 1u : 0u);
        }
        wgmma_commit();
        release_epi_buffer(kb);
        wgmma_wait<0>();   // this k-block's partial is complete and its stage has been read
        wgmma_fence_regs(part);
        if (tid_wg == 0) mbar_arrive(empty_bar(stage));
        if constexpr (kMode != kFp8) {   // acc[4 j + 2 h + e] belongs to row h of the fragment
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            acc[4 * j] = fmaf(part[4 * j], s0, acc[4 * j]);
            acc[4 * j + 1] = fmaf(part[4 * j + 1], s0, acc[4 * j + 1]);
            acc[4 * j + 2] = fmaf(part[4 * j + 2], s1, acc[4 * j + 2]);
            acc[4 * j + 3] = fmaf(part[4 * j + 3], s1, acc[4 * j + 3]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] += part[i];
        }
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      };
      for (int64_t kb = 0; kb < num_k_blocks; ++kb) k_block(kb, std::false_type{});
      if constexpr (kMode == kFp8BlkLora) {
        for (int64_t kb = num_k_blocks; kb < total_k_blocks; ++kb) k_block(kb, std::true_type{});
      }
    } else {
      int prev = 0;
      for (int64_t kb = 0; kb < total_k_blocks; ++kb) {
        mbar_wait_notrace(full_bar(stage), phase);
        const uint64_t da = make_sw128_kmajor_desc(smem_a(stage) + (uint32_t)(cw * 64 * 128));
        const uint64_t db = make_sw128_kmajor_desc(smem_b(stage));
        wgmma_fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k)   // +32 bytes along K per step = +2 in the descriptor's 16-byte units
          Wgmma<BLOCK_N>::mma(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        release_epi_buffer(kb);
        wgmma_wait<1>();   // the group of the previous k-block has retired: its stage may be refilled
        wgmma_fence_regs(acc);
        if (kb > 0 && tid_wg == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (tid_wg == 0) mbar_arrive(empty_bar(prev));   // the tile's last stage: the next tile's k-blocks need it
    }

    if constexpr (lora_mode(kMode)) {
      // DoRA: acc *= col_scale[n] (kLora: passed in the w_scale slot) before the epilogue adds the bias.  A thread's columns are
      // the same for both of its rows, so each scale pair is loaded once per tile.  x * 1.0f is exact: an all-ones scale
      // leaves the accumulator's bits as they are.  Columns >= N are never stored, so their index is clamped instead of
      // branched around: the loads carry no control dependence and can all be in flight at once.
      const float* col_scale = kMode == kLora ? w_scale : fb.col_scale;
      if (col_scale != nullptr) {
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int64_t n = min(n_blk * BLOCK_N + 8 * j + c_frag, p.N - 2);
          const float2 cs = __ldg(reinterpret_cast<const float2*>(col_scale + n));
          acc[4 * j] *= cs.x;
          acc[4 * j + 1] *= cs.y;
          acc[4 * j + 2] *= cs.x;
          acc[4 * j + 3] *= cs.y;
        }
      }
    }

    if constexpr ((kMode == kFp8Blk || kMode == kFp8BlkLora) && BLOCK_N == 128) {
      if (p.epilogue == OSB_EPI_BIAS_GELU_TANH_FP8) {
        // ===================== epilogue: GELU-tanh -> e4m3 codes + one scale per (row, 128 columns) =====================
        // N % 128 == 0 (host check): every column of the tile exists.  Rows >= M take part in the quad shuffles (all lanes
        // must) and store nothing.
        const int64_t n0 = n_blk * BLOCK_N + c_frag;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t row = m_blk * kBlockM + r_frag + 8 * h;
          float amax = 0.f;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int64_t n = n0 + 8 * j;
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if constexpr (kMode == kFp8Blk) {   // kFp8BlkLora: w_scale is already in the accumulator
              const float2 sw = __ldg(reinterpret_cast<const float2*>(w_scale + n));
              v0 *= sw.x;
              v1 *= sw.y;
            }
            if (p.bias) {
              const float2 b = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(p.bias + n)));
              v0 += b.x;
              v1 += b.y;
            }
            v0 = gelu_tanh(v0);
            v1 = gelu_tanh(v1);
            acc[4 * j + 2 * h] = v0;
            acc[4 * j + 2 * h + 1] = v1;
            amax = fmaxf(amax, fmaxf(fabsf(v0), fabsf(v1)));
          }
          amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
          amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
          const float s = amax > 0.f ? amax / 448.0f : 1.0f;
          if (row < p.M) {
            uint8_t* drow = fb.d8 + row * fb.ldd8;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j)   // x / s, IEEE division as the contract states it
              *reinterpret_cast<uint16_t*>(drow + n0 + 8 * j) =
                  (uint16_t)e4m3x2(acc[4 * j + 2 * h] / s, acc[4 * j + 2 * h + 1] / s);
            if (c_frag == 0) fb.d_scale[row * fb.ld_dscale + n_blk] = s;
          }
        }
        continue;
      }
    }

    if constexpr (kMode == kHeadTiles) {
      // ===================== epilogue: head tiles =====================
      // a row's D columns of one head are spread over the 4 lanes of a quad: RMSNorm reduces over the quad,
      // RoPE pairs (2i, 2i+1) sit in one thread.  The stores go out as whole 16-byte units (below), so every lane of a
      // warp takes part in the quad exchanges and only the stores of rows >= M are skipped.
      constexpr int D = BLOCK_N / 2;
      using HT = HeadTileCfg<D>;
      constexpr int JH = D / 8;   // 8-column fragments per head
      const int C = ht.heads * D;
      const uint32_t chunk_bytes = (uint32_t)ht.map.TR * 128u;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = m_blk * kBlockM + r_frag + 8 * h;
        const bool row_ok = row < p.M;
        // token row -> (tile, position in its sequence, row in tile)  (the host checks M < 2^31)
        uint32_t pos = 0, tile_i = 0;
        int r = 0;
        if (row_ok) tile_of_row(ht.map, (uint32_t)row, tile_i, pos, r);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int64_t col0 = n_blk * BLOCK_N + hh * D;
          if (col0 >= p.N) continue;   // uniform over the CTA
          const int kidx = (int)((uint32_t)col0 / (uint32_t)C);
          const int head = (int)((uint32_t)col0 - (uint32_t)kidx * (uint32_t)C) / D;
          const int kind = kidx % ht.nkinds;
          float x[JH][2];
#pragma unroll
          for (int j = 0; j < JH; ++j) {
            x[j][0] = acc[4 * (hh * JH + j) + 2 * h];
            x[j][1] = acc[4 * (hh * JH + j) + 2 * h + 1];
            if (p.bias) {
              const float2 b = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(p.bias + col0 + 8 * j + c_frag)));
              x[j][0] += b.x;
              x[j][1] += b.y;
            }
          }
          if ((ht.norm_mask >> kind) & 1u) {
            float ss = 0.f;
#pragma unroll
            for (int j = 0; j < JH; ++j) ss += x[j][0] * x[j][0] + x[j][1] * x[j][1];
            ss += __shfl_xor_sync(0xffffffffu, ss, 1);
            ss += __shfl_xor_sync(0xffffffffu, ss, 2);
            const float rs = rsqrtf(ss * (1.0f / D) + ht.eps);
            // (a runtime index into the parameter struct would move the whole struct to local memory)
            const __nv_bfloat16* w = kind == 0 ? ht.norm_w[0] : (kind == 1 ? ht.norm_w[1] : (kind == 2 ? ht.norm_w[2] : ht.norm_w[3]));
#pragma unroll
            for (int j = 0; j < JH; ++j) {
              const float2 f = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(w + 8 * j + c_frag)));
              x[j][0] *= rs * f.x;
              x[j][1] *= rs * f.y;
            }
          }
          if ((ht.rope_mask >> kind) & 1u) {   // rows >= M: position 0, never stored
#pragma unroll
            for (int j = 0; j < JH; ++j) {
              const int64_t i = (int64_t)pos * (D / 2) + (8 * j + c_frag) / 2;
              const float cc = __ldg(ht.cos + i), sn = __ldg(ht.sin + i);
              const float a = x[j][0], b = x[j][1];
              x[j][0] = a * cc - b * sn;
              x[j][1] = b * cc + a * sn;
            }
          }
          uint8_t* dst = ht.base + (int64_t)kidx * ht.kind_stride + (int64_t)head * ht.head_stride + (int64_t)tile_i * ht.tile_bytes;
          // Swizzled units, four at a time: lane q of the quad holds columns (2q, 2q + 1) of each of units j0 .. j0 + 3;
          // a 4 x 4 transpose over the quad (two exchange rounds) leaves it all 16 bytes of unit j0 + q.  A warp then
          // writes 64 contiguous bytes of each of its 8 rows per store (four units of one 128-byte swizzle row), where
          // 4-byte stores wrote 16 bytes per row and store.
          const bool odd = (lane & 1) != 0, high = (lane & 2) != 0;
#pragma unroll
          for (int j0 = 0; j0 < HT::MAIN * 8; j0 += 4) {
            uint32_t u0 = pack_bf16x2(x[j0][0], x[j0][1]), u1 = pack_bf16x2(x[j0 + 1][0], x[j0 + 1][1]);
            uint32_t u2 = pack_bf16x2(x[j0 + 2][0], x[j0 + 2][1]), u3 = pack_bf16x2(x[j0 + 3][0], x[j0 + 3][1]);
            uint32_t s0 = __shfl_xor_sync(0xffffffffu, odd ? u0 : u1, 1);   // lanes q, q ^ 1: 2 x 2 blocks
            uint32_t s1 = __shfl_xor_sync(0xffffffffu, odd ? u2 : u3, 1);
            if (odd) { u0 = s0; u2 = s1; } else { u1 = s0; u3 = s1; }
            s0 = __shfl_xor_sync(0xffffffffu, high ? u0 : u2, 2);            // lanes q, q ^ 2: the blocks
            s1 = __shfl_xor_sync(0xffffffffu, high ? u1 : u3, 2);
            if (high) { u0 = s0; u1 = s1; } else { u2 = s0; u3 = s1; }
            if (row_ok)
              *reinterpret_cast<uint4*>(dst + tile_unit_off<HT::MAIN>(r, j0 + (lane & 3), chunk_bytes)) = make_uint4(u0, u1, u2, u3);
          }
          if (!row_ok) continue;
#pragma unroll
          for (int j = HT::MAIN * 8; j < JH; ++j)   // the head-dim tail (core-matrix layout)
            *reinterpret_cast<uint32_t*>(dst + tile_unit_off<HT::MAIN>(r, j, chunk_bytes) + c_frag * 2) = pack_bf16x2(x[j][0], x[j][1]);
          if constexpr (HT::UP > HT::U)   // head-dim padding columns stay zero
            *reinterpret_cast<uint32_t*>(dst + tile_unit_off<HT::MAIN>(r, HT::U, chunk_bytes) + c_frag * 2) = 0u;
        }
      }
    } else if constexpr (kMode == kText) {
      // ===================== epilogue: gated GELU / bias + quick GELU =====================
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = m_blk * kBlockM + r_frag + 8 * h;
        if (row >= p.M) continue;
        __nv_bfloat16* drow = p.D + row * p.ldd;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int64_t n = n_blk * BLOCK_N + 8 * j + c_frag;
          if (n >= p.N) continue;
          float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (p.bias) {
            const float2 b = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(p.bias + n)));
            v0 += b.x;
            v1 += b.y;
          }
          if (p.epilogue == OSB_EPI_GATED_GELU) {   // columns (n, n + 1) = (wi_0, wi_1) of output column n / 2
            drow[n >> 1] = __float2bfloat16_rn(gelu_tanh(v0) * v1);
          } else {                                  // x * sigmoid(1.702 x)
            v0 = v0 / (1.0f + __expf(-1.702f * v0));
            v1 = v1 / (1.0f + __expf(-1.702f * v1));
            *reinterpret_cast<uint32_t*>(drow + n) = pack_bf16x2(v0, v1);
          }
        }
      }
    } else {
      // ===================== staged epilogue: bias / GELU / gate + residual =====================
      // The tile is assembled in the epilogue buffer and leaves by TMA: the buffer row of tile row li is li (for kConv the
      // 5-D output box orders its 128 positions exactly like the A box, so li is also its row there), column c of the tile
      // sits in box c / 64 at 16-byte chunk (c % 64) / 8 XOR (li % 8) - the 128-byte swizzle.  A quad's four lanes cover
      // one 16-byte chunk of a row and the eight rows of a warp's fragment land in eight different chunks: conflict free.
      // Rows >= M and columns >= N are computed like the others and clipped by the tensor map on the store, so the only
      // global reads left are the per-column bias / scale / gate vectors (clamped indices, no control dependence: they can
      // all be in flight at once) and nothing is read after the first store.  The arithmetic per element is the register
      // epilogue's, in its order and with its roundings (explicit _rn operations: no contraction into an FMA).
      static_assert(kStaged, "every other mode has its own epilogue");
      uint8_t* const epi = smem_raw + (epi_base - smem_u32(smem_raw));
      const bool gate_res = p.epilogue == OSB_EPI_BIAS_GATE_RES;
      if (!gate_res) gate_row[0] = gate_row[1] = nullptr;
      const bool has_res = gate_res && p.R != nullptr;
      // With a residual, the producer issued it only after the previous tile's stores had read the buffer; without one,
      // the buffer is free once they have.
      if (p.R != nullptr)
        mbar_wait_notrace(res_bar, it & 1u);
      else if (it > 0)
        mbar_wait_notrace(epi_free, (it - 1) & 1u);
      // One straight-line body per activation, with the optional operands folded into identities that leave every bit of
      // the value as it is (x + -0 = x, x * 1 = x): no branch splits the unrolled loop, so the loads are not held behind one.
      auto body = [&](auto gelu) {
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int64_t n = min(n_blk * BLOCK_N + 8 * j + c_frag, p.N - 2);   // N % 8 == 0: n < N implies n + 1 < N
          float2 sw = make_float2(1.f, 1.f), b = make_float2(-0.f, -0.f);
          if constexpr (kMode == kFp8 || kMode == kFp8Blk) sw = __ldg(reinterpret_cast<const float2*>(w_scale + n));
          if (p.bias) b = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(p.bias + n)));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int li = r_frag + 8 * h;
            uint32_t* const cell = reinterpret_cast<uint32_t*>(epi + (j >> 3) * kEpiBoxBytes + li * 128 +
                                                               (((j & 7) ^ (li & 7)) << 4) + c_frag * 2);
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if constexpr (kMode == kFp8) {
              v0 = __fmul_rn(v0, __fmul_rn(sa[h], sw.x));
              v1 = __fmul_rn(v1, __fmul_rn(sa[h], sw.y));
            } else if constexpr (kMode == kFp8Blk) {   // the A scales are already in the accumulator (kFp8BlkLora: all scales)
              v0 = __fmul_rn(v0, sw.x);
              v1 = __fmul_rn(v1, sw.y);
            }
            v0 = __fadd_rn(v0, b.x);
            v1 = __fadd_rn(v1, b.y);
            if constexpr (decltype(gelu)::value) {
              v0 = gelu_tanh(v0);
              v1 = gelu_tanh(v1);
            } else {
              // the residual element is read before this thread overwrites it with the result
              const float2 g = gate_row[h] ? __ldg(reinterpret_cast<const float2*>(gate_row[h] + n)) : make_float2(1.f, 1.f);
              const float2 rv = has_res ? unpack_bf16x2(*cell) : make_float2(-0.f, -0.f);
              v0 = __fadd_rn(__fmul_rn(v0, g.x), rv.x);
              v1 = __fadd_rn(__fmul_rn(v1, g.y), rv.y);
            }
            *cell = pack_bf16x2(v0, v1);
          }
        }
      };
      if (p.epilogue == OSB_EPI_BIAS_GELU_TANH)
        body(std::true_type{});
      else
        body(std::false_type{});
      // Both consumer warpgroups' writes, made visible to the async proxy, then one thread stores the tile.  It waits only
      // until the stores have READ the buffer (release_epi_buffer in the next tile, or before the CTA exits), which is all
      // the next tile or the CTA's exit needs.  The writes themselves belong to this grid's memory operations, which a
      // dependent kernel's griddepcontrol.wait (PDL) or an ordinary stream-ordered launch waits for in full before it
      // reads the output.
      fence_proxy_async_smem();
      named_barrier_sync(1, 256);
      if (threadIdx.x == 128) {
        const int32_t n0 = (int32_t)(n_blk * BLOCK_N);
        const int live = (int)min((int64_t)(BLOCK_N / 64), (p.N - n0 + 63) / 64);
        for (int c = 0; c < live; ++c) {
          if constexpr (kMode == kConv)
            tma_store_5d(&tmap_d, epi_base + c * kEpiBoxBytes, n0 + 64 * c, tl.w0, tl.h0, tl.t0, tl.n_i);
          else
            tma_store_2d(&tmap_d, epi_base + c * kEpiBoxBytes, n0 + 64 * c, (int32_t)(m_blk * kBlockM));
        }
        bulk_commit_group();
      }
    }
  }
  if constexpr (kStaged) {
    if (threadIdx.x == 128) bulk_wait_group_read_all();   // the last tile's stores have read the buffer: the CTA may exit
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
template <int BLOCK_N, int kMode>
static int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tw, const GemmEpilogueParams& p, const ConvGeom& cg,
                         const HeadTileParams& ht, int64_t tiles, cudaStream_t stream, const CUtensorMap* tu = nullptr,
                         const CUtensorMap* tlb = nullptr, int32_t lora_k_blocks = 0, const float* a_scale = nullptr,
                         const float* w_scale = nullptr, const Fp8BlockParams& fb = Fp8BlockParams{},
                         const CUtensorMap* tr = nullptr, const CUtensorMap* td = nullptr) {
  if (tiles >= (1ll << 31)) { set_error("osb gemm: too many output tiles (%lld)", (long long)tiles); return OSB_ERR_UNSUPPORTED; }
  const int64_t grid = tiles < sm_count() ? tiles : sm_count();   // one CTA per SM, each walks its tiles
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)grid), dim3(kNumThreads),
                                         GemmCfg<BLOCK_N, staged_epilogue(kMode)>::SMEM_BYTES, stream, attr);
  // the LoRA maps are read by kLora only, the residual / output maps by the staged epilogue only (the residual map only
  // when p.R is set); where a map is not read the main maps are passed as placeholders
  OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemm_bf16_kernel<BLOCK_N, kMode>, ta, tw, p, cg, ht, tu ? *tu : ta,
                                    tlb ? *tlb : tw, lora_k_blocks, a_scale, w_scale, fb, tr ? *tr : ta, td ? *td : ta));
  count_launch();
  return OSB_OK;
}

// Staged epilogue maps over the output D and the residual R (when p.R is set; *tr is left unset otherwise): [M, N] with
// the row strides ldd / ldr, boxes of 128 rows x 64 columns.  The extents are exactly M x N, never ldd columns or a
// padded M: the tile stores clip to them, so no byte outside the output view is written.
static int make_epilogue_maps(const GemmEpilogueParams& p, CUtensorMap* tr, CUtensorMap* td) {
  if (int rc = make_tmap_2d_bf16(td, p.D, p.M, p.N, p.ldd, kBlockM, 64)) return rc;
  if (p.R != nullptr) return make_tmap_2d_bf16(tr, p.R, p.M, p.N, p.ldr, kBlockM, 64);
  *tr = *td;
  return OSB_OK;
}

template <int D>
static int launch_gemm_ht(const osb_gemm_args& a, const HeadTileParams& ht, cudaStream_t stream) {
  constexpr int BLOCK_N = 2 * D;   // two heads per tile
  CUtensorMap ta, tw;
  int rc = make_tmap_2d_bf16(&ta, a.A, a.M, a.K, a.lda, kBlockM, kBlockK);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tw, a.W, a.N, a.K, a.ldw, BLOCK_N, kBlockK);
  if (rc) return rc;
  GemmEpilogueParams p = {};
  p.bias = static_cast<const __nv_bfloat16*>(a.bias);
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.group_rows = a.M;
  p.epilogue = OSB_EPI_BIAS;
  const int64_t tiles = ((a.M + kBlockM - 1) / kBlockM) * ((a.N + BLOCK_N - 1) / BLOCK_N);
  ConvGeom cg = {};
  return launch_kernel<BLOCK_N, kHeadTiles>(ta, tw, p, cg, ht, tiles, stream);
}

template <int BLOCK_N>
static int launch_gemm(const osb_gemm_args& a, bool has_res, cudaStream_t stream, const osb_lora_args* lora = nullptr) {
  CUtensorMap ta, tw;
  int rc = make_tmap_2d_bf16(&ta, a.A, a.M, a.K, a.lda, kBlockM, kBlockK);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tw, a.W, a.N, a.K, a.ldw, BLOCK_N, kBlockK);
  if (rc) return rc;
  GemmEpilogueParams p = {};
  p.bias = static_cast<const __nv_bfloat16*>(a.bias);
  p.D = static_cast<__nv_bfloat16*>(a.D);
  p.R = has_res ? static_cast<const __nv_bfloat16*>(a.R) : nullptr;
  p.gate = a.gate;
  p.mod_index = a.mod_index;
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.ldd = a.ldd;
  p.ldr = a.ldr;
  p.group_rows = a.group_rows > 0 ? a.group_rows : a.M;
  p.gate_stride = a.gate_stride;
  p.epilogue = a.epilogue;
  const int64_t tiles = ((a.M + kBlockM - 1) / kBlockM) * ((a.N + BLOCK_N - 1) / BLOCK_N);
  ConvGeom cg = {};
  HeadTileParams ht = {};
  if (lora == nullptr && a.epilogue >= OSB_EPI_GATED_GELU) return launch_kernel<BLOCK_N, kText>(ta, tw, p, cg, ht, tiles, stream);
  CUtensorMap tr, td;
  if ((rc = make_epilogue_maps(p, &tr, &td))) return rc;
  if (lora == nullptr)
    return launch_kernel<BLOCK_N, kPlain>(ta, tw, p, cg, ht, tiles, stream, nullptr, nullptr, 0, nullptr, nullptr,
                                          Fp8BlockParams{}, &tr, &td);
  CUtensorMap tu, tlb;
  if ((rc = make_tmap_2d_bf16(&tu, lora->U, a.M, lora->r, lora->ldu, kBlockM, kBlockK))) return rc;
  if ((rc = make_tmap_2d_bf16(&tlb, lora->B, a.N, lora->r, lora->ldb, BLOCK_N, kBlockK))) return rc;
  return launch_kernel<BLOCK_N, kLora>(ta, tw, p, cg, ht, tiles, stream, &tu, &tlb, (lora->r + kBlockK - 1) / kBlockK,
                                       nullptr, lora->col_scale, Fp8BlockParams{}, &tr, &td);
}

template <int BLOCK_N, int kMode>
static int init_one() {
  OSB_CHECK_CUDA(cudaFuncSetAttribute(gemm_bf16_kernel<BLOCK_N, kMode>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      GemmCfg<BLOCK_N, staged_epilogue(kMode)>::SMEM_BYTES));
  return OSB_OK;
}

int gemm_init() {
  int rc = 0;
  if ((rc = init_one<128, kHeadTiles>())) return rc;
  if ((rc = init_one<144, kHeadTiles>())) return rc;
  if ((rc = init_one<256, kHeadTiles>())) return rc;
  if ((rc = init_one<64, kPlain>())) return rc;
  if ((rc = init_one<128, kPlain>())) return rc;
  if ((rc = init_one<192, kPlain>())) return rc;
  if ((rc = init_one<256, kPlain>())) return rc;
  if ((rc = init_one<64, kConv>())) return rc;
  if ((rc = init_one<128, kConv>())) return rc;
  if ((rc = init_one<192, kConv>())) return rc;
  if ((rc = init_one<256, kConv>())) return rc;
  if ((rc = init_one<64, kLora>())) return rc;
  if ((rc = init_one<128, kLora>())) return rc;
  if ((rc = init_one<192, kLora>())) return rc;
  if ((rc = init_one<256, kLora>())) return rc;
  if ((rc = init_one<64, kText>())) return rc;
  if ((rc = init_one<128, kText>())) return rc;
  if ((rc = init_one<192, kText>())) return rc;
  if ((rc = init_one<256, kText>())) return rc;
  if ((rc = init_one<64, kFp8>())) return rc;
  if ((rc = init_one<128, kFp8>())) return rc;
  if ((rc = init_one<64, kFp8Blk>())) return rc;
  if ((rc = init_one<128, kFp8Blk>())) return rc;
  if ((rc = init_one<64, kFp8BlkLora>())) return rc;
  if ((rc = init_one<128, kFp8BlkLora>())) return rc;
  return OSB_OK;
}

// Tile width: fewest (tiles per CTA, rounded up) x (tile width + 16), i.e. the least padded work once the last round of
// tiles is counted as full, plus what every tile pays besides its main loop (the epilogue, which no main loop hides),
// about 16 columns' worth on one H100 (DESIGN.md 5b); ties go to the wider tile, which re-reads A less often.
static int pick_block_n(int64_t M, int64_t N) {
  if (N <= 64) return 64;
  const int cands[3] = {256, 192, 128};
  int best = 256;
  int64_t best_cost = INT64_MAX;
  for (int i = 0; i < 3; ++i) {
    const int bn = cands[i];
    const int64_t tiles = ((M + kBlockM - 1) / kBlockM) * ((N + bn - 1) / bn);
    const int64_t waves = (tiles + sm_count() - 1) / sm_count();
    const int64_t cost = waves * (bn + 16);
    if (cost < best_cost) { best_cost = cost; best = bn; }
  }
  return best;
}

template <int BLOCK_N, int kMode = kFp8>
static int launch_gemm_fp8(const osb_gemm_fp8_args& a, cudaStream_t stream, const Fp8BlockParams& fb = Fp8BlockParams{},
                           const osb_lora_args* lora = nullptr) {
  CUtensorMap ta, tw;
  int rc = make_tmap_2d_e4m3(&ta, a.A, a.M, a.K, a.lda, kBlockM, 2 * kBlockK);
  if (rc) return rc;
  rc = make_tmap_2d_e4m3(&tw, a.W, a.N, a.K, a.ldw, BLOCK_N, 2 * kBlockK);
  if (rc) return rc;
  GemmEpilogueParams p = {};
  p.bias = static_cast<const __nv_bfloat16*>(a.bias);
  p.D = static_cast<__nv_bfloat16*>(a.D);
  p.R = a.epilogue == OSB_EPI_BIAS_GATE_RES ? static_cast<const __nv_bfloat16*>(a.R) : nullptr;
  p.gate = a.gate;
  p.mod_index = a.mod_index;
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.ldd = a.ldd;
  p.ldr = a.ldr;
  p.group_rows = a.group_rows > 0 ? a.group_rows : a.M;
  p.gate_stride = a.gate_stride;
  p.epilogue = a.epilogue;
  const int64_t tiles = ((a.M + kBlockM - 1) / kBlockM) * ((a.N + BLOCK_N - 1) / BLOCK_N);
  ConvGeom cg = {};
  HeadTileParams ht = {};
  CUtensorMap tr = ta, td = ta;   // the FP8-emitting GELU epilogue writes no bf16 D (it may be null)
  if (a.epilogue != OSB_EPI_BIAS_GELU_TANH_FP8 && (rc = make_epilogue_maps(p, &tr, &td))) return rc;
  if constexpr (kMode == kFp8BlkLora) {
    CUtensorMap tu, tlb;
    if ((rc = make_tmap_2d_bf16(&tu, lora->U, a.M, lora->r, lora->ldu, kBlockM, kBlockK))) return rc;
    if ((rc = make_tmap_2d_bf16(&tlb, lora->B, a.N, lora->r, lora->ldb, BLOCK_N, kBlockK))) return rc;
    return launch_kernel<BLOCK_N, kMode>(ta, tw, p, cg, ht, tiles, stream, &tu, &tlb, (lora->r + kBlockK - 1) / kBlockK,
                                         a.a_scale, a.w_scale, fb, &tr, &td);
  }
  return launch_kernel<BLOCK_N, kMode>(ta, tw, p, cg, ht, tiles, stream, nullptr, nullptr, 0, a.a_scale, a.w_scale, fb,
                                       &tr, &td);
}

// ------------------------------------------------------------------------------------------
// causal 3D convolution as implicit GEMM (NDHWC, input already replicate-padded by osb_vae_prep)
// ------------------------------------------------------------------------------------------
template <int BLOCK_N>
static int launch_conv(const osb_conv3d_args& a, const ConvGeom& cg, const uint32_t box[5], cudaStream_t stream) {
  CUtensorMap ta, tw;
  const uint64_t cp = a.cp;
  // narrow mode: overlapping windows of 64 contiguous elements starting at every w (stride Cp elements): (kw, c) folded
  const uint64_t dims[5] = {a.narrow ? 64 : cp, (uint64_t)a.wp, (uint64_t)a.hp, (uint64_t)a.tp, (uint64_t)a.nb};
  const uint64_t str[4] = {cp * 2, (uint64_t)a.wp * cp * 2, (uint64_t)a.hp * a.wp * cp * 2,
                           (uint64_t)a.tp * a.hp * a.wp * cp * 2};
  const uint32_t es[5] = {1, (uint32_t)a.sw, (uint32_t)a.sh, (uint32_t)a.st, 1};
  int rc = make_tmap_5d_bf16(&ta, a.x_pad, dims, str, box, es);
  if (rc) return rc;
  const int64_t K = (int64_t)(a.narrow ? a.kt * a.kh : a.kt * a.kh * a.kw * (a.cp / 64)) * 64;
  rc = make_tmap_2d_bf16(&tw, a.w, a.cout, K, K, BLOCK_N, kBlockK);
  if (rc) return rc;
  GemmEpilogueParams p = {};
  p.bias = static_cast<const __nv_bfloat16*>(a.bias);
  p.D = static_cast<__nv_bfloat16*>(a.y);
  p.R = static_cast<const __nv_bfloat16*>(a.residual);
  p.M = (int64_t)a.nb * a.t_out * a.h_out * a.w_out;
  p.N = a.cout;
  p.K = K;
  p.ldd = a.cout;
  p.ldr = a.cout;
  p.group_rows = p.M;
  p.epilogue = a.residual ? OSB_EPI_BIAS_GATE_RES : OSB_EPI_BIAS;
  const int64_t tiles = (int64_t)cg.nb * cg.tiles_t * cg.tiles_h * cg.tiles_w * ((a.cout + BLOCK_N - 1) / BLOCK_N);
  HeadTileParams ht = {};
  // output and residual: the NDHWC [nb, t_out, h_out, w_out, cout] tensor, one box = the CTA's Wt x Ht x Tt positions x
  // 64 channels, ordered like the A box (its 128 rows); boxes past the output's edges are clipped on store
  const uint64_t cout = (uint64_t)a.cout;
  const uint64_t odims[5] = {cout, (uint64_t)a.w_out, (uint64_t)a.h_out, (uint64_t)a.t_out, (uint64_t)a.nb};
  const uint64_t ostr[4] = {cout * 2, (uint64_t)a.w_out * cout * 2, (uint64_t)a.h_out * a.w_out * cout * 2,
                            (uint64_t)a.t_out * a.h_out * a.w_out * cout * 2};
  const uint32_t obox[5] = {64, 1u << cg.wt_log2, 1u << cg.ht_log2, 128u >> (cg.wt_log2 + cg.ht_log2), 1};
  const uint32_t ones[5] = {1, 1, 1, 1, 1};
  CUtensorMap tr, td;
  if ((rc = make_tmap_5d_bf16(&td, a.y, odims, ostr, obox, ones))) return rc;
  tr = td;
  if (a.residual && (rc = make_tmap_5d_bf16(&tr, a.residual, odims, ostr, obox, ones))) return rc;
  return launch_kernel<BLOCK_N, kConv>(ta, tw, p, cg, ht, tiles, stream, nullptr, nullptr, 0, nullptr, nullptr,
                                       Fp8BlockParams{}, &tr, &td);
}

}  // namespace osb

namespace osb {

// The adapter operands of osb_gemm_lora and osb_gemm_fp8_lora (`fn` names the entry point in errors).
static int check_lora_args(const char* fn, const osb_lora_args& l) {
  OSB_REQUIRE(l.U && l.B, "%s: null U or B", fn);
  OSB_REQUIRE(l.r > 0 && l.r % 8 == 0, "%s: rank r must be a positive multiple of 8 (zero-pad A and B), got %d", fn, l.r);
  OSB_REQUIRE(l.ldu >= l.r && l.ldb >= l.r && l.ldu % 8 == 0 && l.ldb % 8 == 0 &&
              ((reinterpret_cast<uintptr_t>(l.U) | reinterpret_cast<uintptr_t>(l.B)) & 15) == 0,
              "%s: U and B must be 16-byte aligned with ldu, ldb >= r and multiples of 8 (r %d ldu %lld ldb %lld)", fn,
              l.r, (long long)l.ldu, (long long)l.ldb);
  OSB_REQUIRE((reinterpret_cast<uintptr_t>(l.col_scale) & 7) == 0, "%s: col_scale must be 8-byte aligned", fn);
  return OSB_OK;
}

// Argument checks and tile-width dispatch shared by osb_gemm_bf16 and osb_gemm_lora (`fn` names the entry point in errors).
static int gemm_dispatch(const char* fn, const osb_gemm_args* args, const osb_lora_args* lora, void* stream) {
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(args != nullptr, "%s: null args", fn);
  const osb_gemm_args& a = *args;
  OSB_REQUIRE(a.A && a.W && a.D, "%s: null operand", fn);
  OSB_REQUIRE(a.M > 0 && a.N > 0 && a.K > 0, "%s: empty problem (M %lld N %lld K %lld)", fn,
              (long long)a.M, (long long)a.N, (long long)a.K);
  OSB_REQUIRE(a.K % 8 == 0 && a.N % 8 == 0, "%s: K and N must be multiples of 8 (K %lld N %lld)", fn,
              (long long)a.K, (long long)a.N);
  OSB_REQUIRE(a.ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(a.D) & 15) == 0,
              "%s: D must be 16-byte aligned with ldd %% 8 == 0", fn);
  OSB_REQUIRE(a.epilogue >= OSB_EPI_BIAS && a.epilogue <= OSB_EPI_BIAS_QUICK_GELU,
              "%s: unknown epilogue %d", fn, a.epilogue);
  OSB_REQUIRE(lora == nullptr || a.epilogue <= OSB_EPI_BIAS_GATE_RES,
              "%s: epilogue %d is not built with a LoRA update", fn, a.epilogue);
  if (a.epilogue == OSB_EPI_BIAS_GATE_RES) {
    OSB_REQUIRE(a.R == nullptr || (a.ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(a.R) & 15) == 0),
                "%s: R must be 16-byte aligned with ldr %% 8 == 0", fn);
    OSB_REQUIRE(a.gate == nullptr || (a.gate_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(a.gate) & 15) == 0),
                "%s: gate must be 16-byte aligned with gate_stride %% 4 == 0", fn);
  }
  OSB_REQUIRE(a.bias == nullptr || (reinterpret_cast<uintptr_t>(a.bias) & 15) == 0,
              "%s: bias must be 16-byte aligned", fn);
  OSB_REQUIRE(a.cta_group >= 0 && a.cta_group <= 2, "%s: cta_group must be 0, 1 or 2", fn);
  if (lora != nullptr) {
    if (int rc = check_lora_args(fn, *lora)) return rc;
  }
  const bool has_res = (a.epilogue == OSB_EPI_BIAS_GATE_RES) && a.R != nullptr;
  const int bn = a.block_n ? a.block_n : pick_block_n(a.M, a.N);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (bn == 64) return launch_gemm<64>(a, has_res, s, lora);
  if (bn == 128) return launch_gemm<128>(a, has_res, s, lora);
  if (bn == 192) return launch_gemm<192>(a, has_res, s, lora);
  if (bn == 256) return launch_gemm<256>(a, has_res, s, lora);
  set_error("%s: unsupported block_n %d", fn, bn);
  return OSB_ERR_UNSUPPORTED;
}

}  // namespace osb

extern "C" int osb_gemm_bf16(const osb_gemm_args* args, void* stream) {
  return osb::gemm_dispatch("osb_gemm_bf16", args, nullptr, stream);
}

extern "C" int osb_gemm_lora(const osb_gemm_args* gemm, const osb_lora_args* lora, void* stream) {
  if (lora == nullptr) { osb::set_error("osb_gemm_lora: null lora args"); return OSB_ERR_INVALID; }
  return osb::gemm_dispatch("osb_gemm_lora", gemm, lora, stream);
}

namespace osb {

// Argument checks shared by osb_gemm_fp8 and osb_gemm_fp8_blocks (`fn` names the entry point in errors); fp8_out: the
// FP8-emitting epilogue, whose output is checked by the caller instead of D.
static int check_fp8_args(const char* fn, const osb_gemm_fp8_args* args, bool fp8_out) {
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(args != nullptr, "%s: null args", fn);
  const osb_gemm_fp8_args& a = *args;
  OSB_REQUIRE(a.A && a.W && (a.D || fp8_out) && a.a_scale && a.w_scale, "%s: null operand or scale", fn);
  OSB_REQUIRE(a.M > 0 && a.N > 0 && a.K > 0, "%s: empty problem (M %lld N %lld K %lld)", fn,
              (long long)a.M, (long long)a.N, (long long)a.K);
  OSB_REQUIRE(a.K % 128 == 0, "%s: K must be a multiple of 128 (one e4m3 k-block), got %lld", fn, (long long)a.K);
  OSB_REQUIRE(a.N % 8 == 0, "%s: N must be a multiple of 8, got %lld", fn, (long long)a.N);
  OSB_REQUIRE(a.lda % 16 == 0 && a.ldw % 16 == 0 && a.lda >= a.K && a.ldw >= a.K,
              "%s: lda and ldw must be >= K and multiples of 16 (lda %lld ldw %lld)", fn, (long long)a.lda,
              (long long)a.ldw);
  if (!fp8_out) {
    OSB_REQUIRE(a.ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(a.D) & 15) == 0,
                "%s: D must be 16-byte aligned with ldd %% 8 == 0", fn);
    OSB_REQUIRE(a.epilogue >= OSB_EPI_BIAS && a.epilogue <= OSB_EPI_BIAS_GATE_RES,
                "%s: epilogue %d is not built for FP8 (bias, GELU-tanh, gate + residual)", fn, a.epilogue);
  }
  OSB_REQUIRE((reinterpret_cast<uintptr_t>(a.w_scale) & 7) == 0 && (reinterpret_cast<uintptr_t>(a.a_scale) & 3) == 0,
              "%s: a_scale must be 4-byte and w_scale 8-byte aligned", fn);
  if (a.epilogue == OSB_EPI_BIAS_GATE_RES) {
    OSB_REQUIRE(a.R == nullptr || (a.ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(a.R) & 15) == 0),
                "%s: R must be 16-byte aligned with ldr %% 8 == 0", fn);
    OSB_REQUIRE(a.gate == nullptr || (a.gate_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(a.gate) & 15) == 0),
                "%s: gate must be 16-byte aligned with gate_stride %% 4 == 0", fn);
  }
  OSB_REQUIRE(a.bias == nullptr || (reinterpret_cast<uintptr_t>(a.bias) & 15) == 0, "%s: bias must be 16-byte aligned", fn);
  return OSB_OK;
}

}  // namespace osb

extern "C" int osb_gemm_fp8(const osb_gemm_fp8_args* args, void* stream) {
  using namespace osb;
  if (int rc = check_fp8_args("osb_gemm_fp8", args, false)) return rc;
  const osb_gemm_fp8_args& a = *args;
  // the promoted accumulation holds two accumulators per thread: tiles wider than 128 columns would not fit
  const int bn = a.block_n ? a.block_n : (a.N <= 64 ? 64 : 128);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (bn == 64) return launch_gemm_fp8<64>(a, s);
  if (bn == 128) return launch_gemm_fp8<128>(a, s);
  set_error("osb_gemm_fp8: unsupported block_n %d (64 or 128)", bn);
  return OSB_ERR_UNSUPPORTED;
}

namespace osb {

// osb_gemm_fp8_blocks, and with `lora` osb_gemm_fp8_lora (`fn` names the entry point in errors).
static int fp8_blocks_dispatch(const char* fn, const osb_gemm_fp8_args* args, const osb_fp8_blocks_args* blk,
                               const osb_lora_args* lora, void* stream) {
  const bool fp8_out = args != nullptr && args->epilogue == OSB_EPI_BIAS_GELU_TANH_FP8;
  if (int rc = check_fp8_args(fn, args, fp8_out)) return rc;
  if (lora != nullptr) {
    if (int rc = check_lora_args(fn, *lora)) return rc;
  }
  const osb_gemm_fp8_args& a = *args;
  const osb_fp8_blocks_args& b = *blk;
  OSB_REQUIRE(b.a_scale_ld == 0 || b.a_scale_ld >= a.K / 128,
              "%s: a_scale_ld must be 0 (per-row scales) or >= K / 128 (got %lld, K %lld)", fn,
              (long long)b.a_scale_ld, (long long)a.K);
  int bn = a.block_n ? a.block_n : (a.N <= 64 ? 64 : 128);
  if (fp8_out) {
    // one 128-column output tile = one scale block per row
    OSB_REQUIRE(a.N % 128 == 0, "%s: the FP8 GELU epilogue needs N %% 128 == 0, got %lld", fn, (long long)a.N);
    OSB_REQUIRE(a.block_n == 0 || a.block_n == 128, "%s: the FP8 GELU epilogue needs block_n 128, got %d", fn,
                a.block_n);
    OSB_REQUIRE(b.D8 && b.d_scale, "%s: the FP8 GELU epilogue needs D8 and d_scale", fn);
    OSB_REQUIRE(b.ldd8 >= a.N && b.ldd8 % 2 == 0 && (reinterpret_cast<uintptr_t>(b.D8) & 1) == 0 &&
                b.ld_dscale >= a.N / 128 && (reinterpret_cast<uintptr_t>(b.d_scale) & 3) == 0,
                "%s: D8 must be 2-byte aligned with even ldd8 >= N, d_scale 4-byte aligned with "
                "ld_dscale >= N / 128 (ldd8 %lld ld_dscale %lld)", fn, (long long)b.ldd8, (long long)b.ld_dscale);
    bn = 128;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (lora == nullptr && b.a_scale_ld == 0 && !fp8_out) {   // per-row scales and a bf16 epilogue: exactly osb_gemm_fp8
    if (bn == 64) return launch_gemm_fp8<64>(a, s);
    if (bn == 128) return launch_gemm_fp8<128>(a, s);
  } else {
    Fp8BlockParams fb = {};
    fb.a_ld = b.a_scale_ld ? b.a_scale_ld : 1;
    fb.a_kstride = b.a_scale_ld ? 1 : 0;
    fb.d8 = static_cast<uint8_t*>(b.D8);
    fb.d_scale = b.d_scale;
    fb.ldd8 = b.ldd8;
    fb.ld_dscale = b.ld_dscale;
    if (lora != nullptr) {
      fb.col_scale = lora->col_scale;
      if (bn == 64) return launch_gemm_fp8<64, kFp8BlkLora>(a, s, fb, lora);
      if (bn == 128) return launch_gemm_fp8<128, kFp8BlkLora>(a, s, fb, lora);
    } else {
      if (bn == 64) return launch_gemm_fp8<64, kFp8Blk>(a, s, fb);
      if (bn == 128) return launch_gemm_fp8<128, kFp8Blk>(a, s, fb);
    }
  }
  set_error("%s: unsupported block_n %d (64 or 128)", fn, bn);
  return OSB_ERR_UNSUPPORTED;
}

}  // namespace osb

extern "C" int osb_gemm_fp8_blocks(const osb_gemm_fp8_args* args, const osb_fp8_blocks_args* blk, void* stream) {
  if (blk == nullptr) { osb::set_error("osb_gemm_fp8_blocks: null block args"); return OSB_ERR_INVALID; }
  return osb::fp8_blocks_dispatch("osb_gemm_fp8_blocks", args, blk, nullptr, stream);
}

extern "C" int osb_gemm_fp8_lora(const osb_gemm_fp8_args* args, const osb_fp8_blocks_args* blk,
                                 const osb_lora_args* lora, void* stream) {
  if (blk == nullptr || lora == nullptr) { osb::set_error("osb_gemm_fp8_lora: null block or lora args"); return OSB_ERR_INVALID; }
  return osb::fp8_blocks_dispatch("osb_gemm_fp8_lora", args, blk, lora, stream);
}

extern "C" int osb_conv3d_ndhwc(const osb_conv3d_args* args, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(args != nullptr, "osb_conv3d_ndhwc: null args");
  const osb_conv3d_args& a = *args;
  OSB_REQUIRE(a.x_pad && a.w && a.y, "osb_conv3d_ndhwc: null tensor");
  OSB_REQUIRE(a.nb > 0 && a.t_out > 0 && a.h_out > 0 && a.w_out > 0 && a.cout > 0, "osb_conv3d_ndhwc: empty output");
  OSB_REQUIRE(a.cout % 8 == 0, "osb_conv3d_ndhwc: Cout must be a multiple of 8 (pad the weights), got %d", a.cout);
  OSB_REQUIRE(a.st >= 1 && a.st <= 2 && a.sh >= 1 && a.sh <= 2 && a.sw >= 1 && a.sw <= 2, "osb_conv3d_ndhwc: strides must be 1 or 2");
  OSB_REQUIRE(a.kt >= 1 && a.kh >= 1 && a.kw >= 1 && a.kt <= 3 && a.kh <= 3 && a.kw <= 3, "osb_conv3d_ndhwc: taps must be 1..3");
  if (a.narrow) {
    OSB_REQUIRE((a.cp == 8 || a.cp == 16) && a.kw * a.cp <= 64,
                "osb_conv3d_ndhwc: narrow mode needs Cp in {8,16} with kw*Cp <= 64 (Cp %d kw %d)", a.cp, a.kw);
  } else {
    OSB_REQUIRE(a.cp % 64 == 0, "osb_conv3d_ndhwc: Cp must be a multiple of 64 (or use narrow mode), got %d", a.cp);
  }
  OSB_REQUIRE((a.t_out - 1) * a.st + a.kt <= a.tp && (a.h_out - 1) * a.sh + a.kh <= a.hp && (a.w_out - 1) * a.sw + a.kw <= a.wp,
              "osb_conv3d_ndhwc: padded input [%d,%d,%d] too small for output [%d,%d,%d]", a.tp, a.hp, a.wp, a.t_out,
              a.h_out, a.w_out);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(a.x_pad) | reinterpret_cast<uintptr_t>(a.w) | reinterpret_cast<uintptr_t>(a.y) |
                reinterpret_cast<uintptr_t>(a.bias) | reinterpret_cast<uintptr_t>(a.residual)) & 15) == 0,
              "osb_conv3d_ndhwc: tensors must be 16-byte aligned");

  // box of 128 output positions per CTA: minimise padded work, prefer wide W
  ConvGeom cg = {};
  double best = 1e30;
  for (int wl = 7; wl >= 3; --wl) {
    for (int hl = 0; wl + hl <= 7; ++hl) {
      const int Wt = 1 << wl, Ht = 1 << hl, Tt = 128 >> (wl + hl);
      const int64_t tw = (a.w_out + Wt - 1) / Wt, th = (a.h_out + Ht - 1) / Ht, tt = (a.t_out + Tt - 1) / Tt;
      const double work = (double)(tw * Wt) * (double)(th * Ht) * (double)(tt * Tt);
      if (work < best * 0.999) {
        best = work;
        cg.wt_log2 = wl; cg.ht_log2 = hl;
        cg.tiles_w = (int)tw; cg.tiles_h = (int)th; cg.tiles_t = (int)tt;
      }
    }
  }
  cg.nb = a.nb;
  cg.w_out = a.w_out; cg.h_out = a.h_out; cg.t_out = a.t_out;
  cg.sw = a.sw; cg.sh = a.sh; cg.st = a.st;
  cg.kw_n = a.narrow ? 1 : a.kw; cg.kh_n = a.kh;
  cg.cin_chunks = a.narrow ? 1 : a.cp / 64;
  const uint32_t box[5] = {64, (uint32_t)((1 << cg.wt_log2) * a.sw), (uint32_t)((1 << cg.ht_log2) * a.sh),
                           (uint32_t)((128 >> (cg.wt_log2 + cg.ht_log2)) * a.st), 1};
  int bn = a.block_n;
  if (bn == 0) bn = a.cout <= 64 ? 64 : (a.cout <= 128 ? 128 : (a.cout % 256 == 0 ? 256 : (a.cout % 192 == 0 ? 192 : 256)));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (bn == 64) return launch_conv<64>(a, cg, box, s);
  if (bn == 128) return launch_conv<128>(a, cg, box, s);
  if (bn == 192) return launch_conv<192>(a, cg, box, s);
  if (bn == 256) return launch_conv<256>(a, cg, box, s);
  set_error("osb_conv3d_ndhwc: unsupported block_n %d", bn);
  return OSB_ERR_UNSUPPORTED;
}

extern "C" int osb_gemm_head_tiles(const osb_gemm_args* args, const osb_head_tiles_args* targs, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(args != nullptr && targs != nullptr, "osb_gemm_head_tiles: null args");
  const osb_gemm_args& a = *args;
  const osb_head_tiles_args& t = *targs;
  OSB_REQUIRE(a.A && a.W && t.tiles, "osb_gemm_head_tiles: null operand");
  OSB_REQUIRE(a.M > 0 && a.M < (1ll << 31) && a.N > 0 && a.N < (1ll << 31) && a.K > 0 && a.K % 8 == 0, "osb_gemm_head_tiles: bad problem (M %lld N %lld K %lld)",
              (long long)a.M, (long long)a.N, (long long)a.K);
  const int D = t.head_dim;
  OSB_REQUIRE(D == 64 || D == 72 || D == 128, "osb_gemm_head_tiles: head_dim %d not built (64, 72, 128)", D);
  OSB_REQUIRE(t.num_heads > 0 && t.num_heads % 2 == 0 && a.N % ((int64_t)t.num_heads * D) == 0,
              "osb_gemm_head_tiles: N (%lld) must be a multiple of num_heads*head_dim with an even head count (%d x %d)",
              (long long)a.N, t.num_heads, D);
  OSB_REQUIRE(t.nkinds >= 1 && t.nkinds <= 4, "osb_gemm_head_tiles: nkinds must be 1..4");
  const osb_tile_map& m = t.map;
  HeadTileParams ht = {};
  const int rc = make_tile_map(&ht.map, m, "osb_gemm_head_tiles");
  if (rc) return rc;
  OSB_REQUIRE(a.M % (m.mode == 0 ? m.L : (int64_t)m.S * m.T) == 0,
              "osb_gemm_head_tiles: M (%lld) is not a whole number of sequences", (long long)a.M);
  OSB_REQUIRE((reinterpret_cast<uintptr_t>(t.tiles) & 15) == 0 && t.kind_stride % 16 == 0 && t.head_stride % 16 == 0,
              "osb_gemm_head_tiles: tile buffer must be 16-byte aligned");
  OSB_REQUIRE(a.bias == nullptr || (reinterpret_cast<uintptr_t>(a.bias) & 15) == 0, "osb_gemm_head_tiles: bias must be 16-byte aligned");
  const int dp = (D + 15) / 16 * 16;
  const int64_t tile_bytes = (int64_t)m.tile_rows * dp * 2;
  const int64_t tph = osb_head_tiles_per_head(&m, a.M);
  OSB_REQUIRE(t.head_stride >= tph * tile_bytes, "osb_gemm_head_tiles: head_stride %lld < %lld tiles of %lld bytes",
              (long long)t.head_stride, (long long)tph, (long long)tile_bytes);
  OSB_REQUIRE(tph < (1ll << 31), "osb_gemm_head_tiles: too many tiles");
  ht.base = static_cast<uint8_t*>(t.tiles);
  ht.kind_stride = t.kind_stride; ht.head_stride = t.head_stride;
  ht.tile_bytes = (int32_t)tile_bytes;
  ht.heads = t.num_heads; ht.nkinds = t.nkinds;
  ht.norm_mask = t.norm_mask; ht.rope_mask = t.rope_mask;
  for (int k = 0; k < 4; ++k) {
    ht.norm_w[k] = static_cast<const __nv_bfloat16*>(t.norm_w[k]);
    OSB_REQUIRE(!((t.norm_mask >> k) & 1u) || (k < t.nkinds && t.norm_w[k] != nullptr && (reinterpret_cast<uintptr_t>(t.norm_w[k]) & 15) == 0),
                "osb_gemm_head_tiles: kind %d has RMSNorm enabled but no (16-byte aligned) weight", k);
  }
  ht.eps = t.norm_eps;
  ht.cos = t.rope_cos; ht.sin = t.rope_sin;
  OSB_REQUIRE(t.rope_mask == 0 || (t.rope_cos && t.rope_sin && ((reinterpret_cast<uintptr_t>(t.rope_cos) | reinterpret_cast<uintptr_t>(t.rope_sin)) & 15) == 0),
              "osb_gemm_head_tiles: RoPE enabled but the cos / sin tables are missing or not 16-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (D == 64) return launch_gemm_ht<64>(a, ht, s);
  if (D == 72) return launch_gemm_ht<72>(a, ht, s);
  return launch_gemm_ht<128>(a, ht, s);
}
