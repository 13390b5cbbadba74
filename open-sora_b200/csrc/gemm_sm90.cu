// bf16 GEMM for sm_90a:  D[M,N] = epilogue(A[M,K] * W[N,K]^T + bias)
//
// Warp-specialised kernel, one 128 x BLOCK_N output tile per CTA.  Warpgroup 0 is the producer: one thread streams
// the A and W tiles with TMA into 128-byte-swizzled shared memory (BLOCK_K = 64 bf16 = one swizzle row) through a
// ring of mbarrier-guarded stages.  Warpgroups 1 and 2 each own 64 accumulator rows: wgmma.mma_async reads both
// operands straight from the swizzled tiles (matrix descriptors), the fp32 accumulator lives in registers and the
// epilogue runs on those registers, so the accumulator never goes through memory before its single rounding to bf16.
// One wgmma group stays in flight while the next stage is waited for; a stage is handed back to the producer as soon
// as the group that read it has retired.
//
// The same main loop serves five front ends (template kMode):
//   kPlain      nn.Linear with fused bias / GELU(tanh) / gate * x + residual epilogues;
//   kConv       causal 3D convolution as implicit GEMM: every k-block is ONE 5-D TMA box of the padded NDHWC input;
//   kHeadTiles  q / k / v projection whose epilogue writes per-head operand tiles (tiles.cuh) with RMSNorm + RoPE;
//   kLora       kPlain plus an unmerged low-rank update: after the K loop the producer streams ceil(r / 64) more
//               k-blocks, U = x A^T [M, r] in the A slot and s B [N, r] in the W slot, through the same stage ring, so
//               A W^T + U (s B)^T lands in one fp32 accumulator before the unchanged epilogue.
//   kText       nn.Linear with the text encoders' activations: T5's gated GELU gelu_tanh(x wi_0^T) * (x wi_1^T) over a
//               weight whose rows interleave wi_0 and wi_1 (both halves of an output column sit in one thread's
//               accumulator pair, the [M, 2 d_ff] product never leaves registers), and CLIP's bias + quick GELU.
//
// Replaces every nn.Linear on the denoiser block path of the reference
// (opensora/models/mmdit/layers.py:209-214,247-252,277-281,314-334,401) and the fused epilogues
// replace the separate bias / GELU(tanh) / gate*x+residual elementwise kernels.
#include <stdlib.h>

#include "common.cuh"
#include "tiles.cuh"
#include "wgmma.cuh"

namespace osb {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kNumThreads = 384;            // producer warpgroup + two consumer warpgroups
constexpr int kStageBudget = 200 * 1024;    // operand ring (one CTA per SM; 227 KB is the per-block limit)

enum { kPlain = 0, kConv = 1, kHeadTiles = 2, kLora = 3, kText = 4 };

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
// CTA owns a Tt x Ht x Wt box of output positions (128 rows).  The K loop walks (kt, kh, kw) taps x 64-channel
// chunks; every k-block is ONE 5-D TMA box load at the tap's offset.
struct ConvGeom {
  int32_t wt_log2, ht_log2;              // box: Wt = 1 << wt_log2, Ht = 1 << ht_log2, Tt = 128 / (Wt * Ht)
  int32_t tiles_w, tiles_h, tiles_t, nb; // tiles per dimension, batch
  int32_t w_out, h_out, t_out;
  int32_t sw, sh, st;                    // convolution strides
  int32_t kw_n, kh_n;                    // taps along w, h (taps along t = k-blocks / (kw_n * kh_n * cin_chunks))
  int32_t cin_chunks;                    // 64-wide channel chunks per tap
};

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int A_BYTES = kBlockM * kBlockK * 2;
  static constexpr int B_BYTES = BLOCK_N * kBlockK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES_RAW = kStageBudget / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 6 ? 6 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 2 * 8 * STAGES;  // +1024 alignment slack
  static_assert(STAGES >= 2, "pipeline needs at least two stages");
  static_assert(B_BYTES % 1024 == 0, "W tile must keep 1024-byte swizzle-atom alignment");
  static_assert(BLOCK_N % 16 == 0 && BLOCK_N <= 256, "wgmma N");
};

template <int BLOCK_N, int kMode>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                 const GemmEpilogueParams p, const ConvGeom cg, const HeadTileParams ht,
                 const __grid_constant__ CUtensorMap tmap_u, const __grid_constant__ CUtensorMap tmap_lb,
                 const int32_t lora_k_blocks) {   // kLora only: U / s B maps and ceil(r / 64)
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int kStages = Cfg::STAGES;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 1024-byte aligned
  const uint32_t bar_base = smem_base + kStages * Cfg::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };
  auto smem_a = [&](int s) { return smem_base + s * Cfg::STAGE_BYTES; };
  auto smem_b = [&](int s) { return smem_base + s * Cfg::STAGE_BYTES + Cfg::A_BYTES; };

  const int wg = threadIdx.x >> 7;
  const int tid_wg = threadIdx.x & 127;
  const int64_t num_n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int64_t m_blk = blockIdx.x / num_n_blocks, n_blk = blockIdx.x % num_n_blocks;
  const int64_t num_k_blocks = (p.K + kBlockK - 1) / kBlockK;
  const int64_t total_k_blocks = kMode == kLora ? num_k_blocks + lora_k_blocks : num_k_blocks;
  // conv: m_blk -> (batch, t-tile, h-tile, w-tile); the box origin in OUTPUT coordinates
  int n_i = 0, t0 = 0, h0 = 0, w0 = 0;
  if constexpr (kMode == kConv) {
    const int tw = (int)(m_blk % cg.tiles_w);
    const int th = (int)((m_blk / cg.tiles_w) % cg.tiles_h);
    const int tt = (int)((m_blk / ((int64_t)cg.tiles_w * cg.tiles_h)) % cg.tiles_t);
    n_i = (int)(m_blk / ((int64_t)cg.tiles_w * cg.tiles_h * cg.tiles_t));
    w0 = tw << cg.wt_log2;
    h0 = th << cg.ht_log2;
    t0 = tt * (128 >> (cg.wt_log2 + cg.ht_log2));
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_w);
    if constexpr (kMode == kLora) {
      tma_prefetch_desc(&tmap_u);
      tma_prefetch_desc(&tmap_lb);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel's tail; its outputs are visible from here on

  if (wg == 0) {
    // ===================== TMA producer (A and W tiles) =====================
    if (tid_wg == 0) {
      const int32_t a_row = (int32_t)(m_blk * kBlockM);
      const int32_t w_row = (int32_t)(n_blk * BLOCK_N);
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait_notrace(empty_bar(stage), phase ^ 1);
        const int32_t k0 = (int32_t)(kb * kBlockK);
        mbar_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);   // out-of-bounds box elements are zero filled and counted
        if constexpr (kMode == kConv) {   // tap offsets in the padded input, output origin scaled by the stride
          const int tap = (int)(kb / cg.cin_chunks);
          const int32_t ac = (int32_t)(kb - (int64_t)tap * cg.cin_chunks) * kBlockK;
          const int32_t aw = w0 * cg.sw + tap % cg.kw_n;
          const int32_t ah = h0 * cg.sh + (tap / cg.kw_n) % cg.kh_n;
          const int32_t at = t0 * cg.st + tap / (cg.kw_n * cg.kh_n);
          tma_load_5d(&tmap_a, full_bar(stage), smem_a(stage), ac, aw, ah, at, n_i);
        } else {
          tma_load_2d(&tmap_a, full_bar(stage), smem_a(stage), k0, a_row);
        }
        tma_load_2d(&tmap_w, full_bar(stage), smem_b(stage), k0, w_row);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      if constexpr (kMode == kLora) {   // the rank tail beyond r is zero filled in both U and s B
        for (int32_t lk = 0; lk < lora_k_blocks; ++lk) {
          mbar_wait_notrace(empty_bar(stage), phase ^ 1);
          mbar_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);
          tma_load_2d(&tmap_u, full_bar(stage), smem_a(stage), lk * kBlockK, a_row);
          tma_load_2d(&tmap_lb, full_bar(stage), smem_b(stage), lk * kBlockK, w_row);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
      pdl_launch_dependents();  // all loads issued: dependents may start filling SMs as they are vacated
    }
    return;
  }

  // ===================== consumers: wgmma main loop =====================
  const int cw = wg - 1;   // accumulator rows [64 cw, 64 cw + 64) of the tile
  float acc[BLOCK_N / 2];
#pragma unroll
  for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
  {
    int stage = 0, prev = 0;
    uint32_t phase = 0;
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
      wgmma_wait<1>();   // the group of the previous k-block has retired: its stage may be refilled
      wgmma_fence_regs(acc);
      if (kb > 0 && tid_wg == 0) mbar_arrive(empty_bar(prev));
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
  }

  // accumulator fragment: acc[4 j + 2 h + e] = (row 16 warp + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e)
  const int warp_in = tid_wg >> 5, lane = tid_wg & 31;
  const int r_frag = cw * 64 + warp_in * 16 + (lane >> 2);
  const int c_frag = 2 * (lane & 3);

  if constexpr (kMode == kHeadTiles) {
    // ===================== epilogue: head tiles =====================
    // a row's D columns of one head are spread over the 4 lanes of a quad: RMSNorm reduces over the quad,
    // RoPE pairs (2i, 2i+1) sit in one thread.
    constexpr int D = BLOCK_N / 2;
    using HT = HeadTileCfg<D>;
    constexpr int JH = D / 8;   // 8-column fragments per head
    const int C = ht.heads * D;
    const uint32_t chunk_bytes = (uint32_t)ht.map.TR * 128u;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t row = m_blk * kBlockM + r_frag + 8 * h;
      const bool row_ok = row < p.M;
      // token row -> (position in its sequence, tile, row in tile)  (32-bit arithmetic: the host checks M < 2^31)
      uint32_t pos = 0, tile_i = 0, seq;
      int r = 0;
      if (row_ok) {
        const uint32_t row32 = (uint32_t)row;
        if (ht.map.mode == 0) {
          seq = row32 / (uint32_t)ht.map.L;
          pos = row32 - seq * (uint32_t)ht.map.L;
        } else {
          const uint32_t ts = (uint32_t)ht.map.T * (uint32_t)ht.map.S;
          const uint32_t b = row32 / ts;
          const uint32_t rem = row32 - b * ts;
          pos = rem / (uint32_t)ht.map.S;
          seq = b * (uint32_t)ht.map.S + (rem - pos * (uint32_t)ht.map.S);
        }
        if (ht.map.G > 1) {
          tile_i = seq / (uint32_t)ht.map.G;
          r = (int)((seq - tile_i * (uint32_t)ht.map.G) * (uint32_t)ht.map.L + pos);
        } else {
          const uint32_t jt = pos / (uint32_t)ht.map.TR;
          tile_i = seq * (uint32_t)ht.map.tps + jt;
          r = (int)(pos - jt * (uint32_t)ht.map.TR);
        }
      }
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
        if (!row_ok) continue;
        if ((ht.rope_mask >> kind) & 1u) {
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
#pragma unroll
        for (int j = 0; j < JH; ++j)
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
    // ===================== epilogue: bias / GELU / gate + residual =====================
    const uint32_t group_rows32 = (uint32_t)(p.group_rows > 0xffffffffll ? 0xffffffffu : p.group_rows);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int li = r_frag + 8 * h;   // row inside the tile
      int64_t row = m_blk * kBlockM + li;
      bool row_ok = row < p.M;
      if constexpr (kMode == kConv) {  // box-local row -> (t, h, w) output position -> flattened NDHWC row
        const int w = w0 + (li & ((1 << cg.wt_log2) - 1));
        const int hy = h0 + ((li >> cg.wt_log2) & ((1 << cg.ht_log2) - 1));
        const int t = t0 + (li >> (cg.wt_log2 + cg.ht_log2));
        row_ok = w < cg.w_out && hy < cg.h_out && t < cg.t_out;
        row = (((int64_t)n_i * cg.t_out + t) * cg.h_out + hy) * cg.w_out + w;
      }
      if (!row_ok) continue;
      const float* gate_row = nullptr;
      if ((kMode == kPlain || kMode == kLora) && p.epilogue == OSB_EPI_BIAS_GATE_RES && p.gate != nullptr) {
        int64_t gi = (uint32_t)row / group_rows32;
        if (p.mod_index) gi = p.mod_index[gi];
        gate_row = p.gate + gi * p.gate_stride;
      }
      __nv_bfloat16* drow = p.D + row * p.ldd;
      const __nv_bfloat16* rrow = p.R ? p.R + row * p.ldr : nullptr;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int64_t n = n_blk * BLOCK_N + 8 * j + c_frag;
        if (n >= p.N) continue;   // N % 8 == 0: n < N implies n + 1 < N
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (p.bias) {
          const float2 b = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(p.bias + n)));
          v0 += b.x;
          v1 += b.y;
        }
        if (p.epilogue == OSB_EPI_BIAS_GELU_TANH) {
          v0 = gelu_tanh(v0);
          v1 = gelu_tanh(v1);
        } else if (p.epilogue == OSB_EPI_BIAS_GATE_RES) {
          if (gate_row != nullptr) {
            const float2 g = __ldg(reinterpret_cast<const float2*>(gate_row + n));
            v0 *= g.x;
            v1 *= g.y;
          }
          if (rrow != nullptr) {   // R may alias D: the element is read before this thread overwrites it
            const float2 rv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(rrow + n));
            v0 += rv.x;
            v1 += rv.y;
          }
        }
        *reinterpret_cast<uint32_t*>(drow + n) = pack_bf16x2(v0, v1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
template <int BLOCK_N, int kMode>
static int launch_kernel(const CUtensorMap& ta, const CUtensorMap& tw, const GemmEpilogueParams& p, const ConvGeom& cg,
                         const HeadTileParams& ht, int64_t tiles, cudaStream_t stream, const CUtensorMap* tu = nullptr,
                         const CUtensorMap* tlb = nullptr, int32_t lora_k_blocks = 0) {
  if (tiles >= (1ll << 31)) { set_error("osb gemm: too many output tiles (%lld)", (long long)tiles); return OSB_ERR_UNSUPPORTED; }
  cudaLaunchAttribute attr[2];
  cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)tiles), dim3(kNumThreads), GemmCfg<BLOCK_N>::SMEM_BYTES, stream, attr);
  // the LoRA maps are read by kLora only; every other mode gets the main maps as placeholders
  OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemm_bf16_kernel<BLOCK_N, kMode>, ta, tw, p, cg, ht, tu ? *tu : ta,
                                    tlb ? *tlb : tw, lora_k_blocks));
  count_launch();
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
  if (lora == nullptr) return launch_kernel<BLOCK_N, kPlain>(ta, tw, p, cg, ht, tiles, stream);
  CUtensorMap tu, tlb;
  if ((rc = make_tmap_2d_bf16(&tu, lora->U, a.M, lora->r, lora->ldu, kBlockM, kBlockK))) return rc;
  if ((rc = make_tmap_2d_bf16(&tlb, lora->B, a.N, lora->r, lora->ldb, BLOCK_N, kBlockK))) return rc;
  return launch_kernel<BLOCK_N, kLora>(ta, tw, p, cg, ht, tiles, stream, &tu, &tlb, (lora->r + kBlockK - 1) / kBlockK);
}

template <int BLOCK_N, int kMode>
static int init_one() {
  OSB_CHECK_CUDA(cudaFuncSetAttribute(gemm_bf16_kernel<BLOCK_N, kMode>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      GemmCfg<BLOCK_N>::SMEM_BYTES));
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
  return OSB_OK;
}

// Tile width: fewest (waves of tiles over the SMs) x (tile width), i.e. the least padded work once the last wave
// is counted as full; ties go to the wider tile, which re-reads A less often.
static int pick_block_n(int64_t M, int64_t N) {
  if (N <= 64) return 64;
  const int cands[3] = {256, 192, 128};
  int best = 256;
  int64_t best_cost = INT64_MAX;
  for (int i = 0; i < 3; ++i) {
    const int bn = cands[i];
    const int64_t tiles = ((M + kBlockM - 1) / kBlockM) * ((N + bn - 1) / bn);
    const int64_t waves = (tiles + sm_count() - 1) / sm_count();
    const int64_t cost = waves * bn;
    if (cost < best_cost) { best_cost = cost; best = bn; }
  }
  return best;
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
  return launch_kernel<BLOCK_N, kConv>(ta, tw, p, cg, ht, tiles, stream);
}

}  // namespace osb

namespace osb {

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
    const osb_lora_args& l = *lora;
    OSB_REQUIRE(l.U && l.B, "%s: null U or B", fn);
    OSB_REQUIRE(l.r > 0 && l.r % 8 == 0, "%s: rank r must be a positive multiple of 8 (zero-pad A and B), got %d", fn, l.r);
    OSB_REQUIRE(l.ldu >= l.r && l.ldb >= l.r && l.ldu % 8 == 0 && l.ldb % 8 == 0 &&
                ((reinterpret_cast<uintptr_t>(l.U) | reinterpret_cast<uintptr_t>(l.B)) & 15) == 0,
                "%s: U and B must be 16-byte aligned with ldu, ldb >= r and multiples of 8 (r %d ldu %lld ldb %lld)", fn,
                l.r, (long long)l.ldu, (long long)l.ldb);
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
  OSB_REQUIRE(m.mode == 0 || m.mode == 1, "osb_gemm_head_tiles: unknown tile map mode %d", m.mode);
  OSB_REQUIRE(m.L > 0 && m.G >= 1 && m.tile_rows > 0 && m.tile_rows <= 128 && m.tile_rows % 8 == 0,
              "osb_gemm_head_tiles: bad tile map (L %d G %d rows %d)", m.L, m.G, m.tile_rows);
  OSB_REQUIRE(m.G == 1 ? (m.tps == (m.L + m.tile_rows - 1) / m.tile_rows) : (m.G * m.L <= m.tile_rows && m.tps == 1),
              "osb_gemm_head_tiles: tile map inconsistent (L %d G %d tps %d rows %d)", m.L, m.G, m.tps, m.tile_rows);
  OSB_REQUIRE(m.mode == 0 ? (a.M % m.L == 0) : (m.S > 0 && m.T == m.L && a.M % ((int64_t)m.S * m.T) == 0),
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
  HeadTileParams ht = {};
  ht.base = static_cast<uint8_t*>(t.tiles);
  ht.kind_stride = t.kind_stride; ht.head_stride = t.head_stride;
  ht.map.mode = m.mode; ht.map.L = m.L; ht.map.S = m.S; ht.map.T = m.T; ht.map.G = m.G; ht.map.tps = m.tps; ht.map.TR = m.tile_rows;
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
