// Head tiles: the on-HBM image of a shared-memory attention operand tile for one attention head.
//
// A head tile holds TR <= 128 token rows (TR % 8 == 0) of ONE head, already in the shared-memory layout the attention
// kernel reads (bank-conflict-free ldmatrix rows of 16 bytes), so the kernel moves it with a single 1-D bulk copy
// (cp.async.bulk) and never transforms the data:
//   bytes [0, MAIN * TR * 128)    MAIN = D / 64 chunks of [TR rows x 64 columns] bf16, 128-byte swizzle
//                                 (row r, 16-byte unit u at (r/8)*1024 + (r%8)*128 + ((u ^ r%8) * 16))
//   bytes [.., + TR * 32)         head-dim tail (D % 64 != 0: columns 64*MAIN .. +15, zero padded) in the
//                                 no-swizzle core-matrix layout (8 rows x 16 B; K-adjacent matrices 128 B apart,
//                                 8-row groups 256 B apart)
// The same bytes serve as the operand of S = Q K^T (ldmatrix) and of O = P V (ldmatrix.trans).
// Producers: the head-tile epilogue of gemm_bf16_kernel (bias + per-head RMSNorm + RoPE fused, gemm_sm90.cu) and the
// staging step of attn_short_kernel.  Consumers: attn_tiles_kernel / attn_short_kernel (attn_sm90.cu).
#pragma once

#include "common.cuh"

namespace osb {

template <int D>
struct HeadTileCfg {
  static constexpr int DP = (D + 15) / 16 * 16;   // padded head dim (MMA K of QK^T, N of PV)
  static constexpr int MAIN = D / 64;             // full 64-wide swizzled chunks
  static constexpr int TAIL = DP - MAIN * 64;     // 0 or 16
  static constexpr int U = D / 8;                 // 16-byte units per head row
  static constexpr int UP = DP / 8;
  static constexpr int ROW_BYTES = DP * 2;        // bytes per token row in a tile (160 for D = 72)
  static_assert(TAIL == 0 || TAIL == 16, "head_dim tail must be one MMA K step");
  static_assert(D % 8 == 0, "head_dim must be a multiple of 8");
};

// How GEMM rows (tokens) map to (tile, row in tile); shared by the producing epilogue and by the attention kernel's
// output addressing (the inverse map).
//   mode 0: sequences are contiguous row blocks: seq = row / L, pos = row % L                (spatial, cross, text)
//   mode 1: frame-major token stream viewed along T: row = (b*T + t)*S + s -> seq = b*S + s, pos = t    (temporal)
//   G > 1 : G short sequences packed per tile: tile = seq / G, r = (seq % G) * L + pos              (G * L <= TR)
//   G == 1: tile = seq * tps + pos / TR, r = pos % TR                                       (tps = ceil(L / TR))
struct TileMap {
  int32_t mode, L, S, T, G, tps, TR;
};

__host__ __device__ inline void tile_of_row(const TileMap& m, int64_t row, int64_t& tile, int& r) {
  int64_t seq;
  int pos;
  if (m.mode == 0) {
    seq = row / m.L;
    pos = (int)(row - seq * m.L);
  } else {
    const int64_t ts = (int64_t)m.T * m.S;
    const int64_t b = row / ts;
    const int64_t rem = row - b * ts;
    const int t = (int)(rem / m.S);
    seq = b * m.S + (rem - (int64_t)t * m.S);
    pos = t;
  }
  if (m.G > 1) {
    tile = seq / m.G;
    r = (int)(seq - tile * m.G) * m.L + pos;
  } else {
    const int j = pos / m.TR;
    tile = seq * m.tps + j;
    r = pos - j * m.TR;
  }
}

// inverse: (sequence, position) -> row of the token stream
__host__ __device__ inline int64_t row_of_token(const TileMap& m, int64_t seq, int pos) {
  if (m.mode == 0) return seq * m.L + pos;
  const int64_t b = seq / m.S, s = seq - b * m.S;
  return (b * m.T + pos) * m.S + s;
}

#ifdef __CUDACC__
// byte offset of 16-byte unit `u` (0..7) of row `r` inside a [rows x 64] bf16 SW128 chunk
__device__ __forceinline__ uint32_t sw128_off(int r, int u) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((u ^ (r & 7)) << 4));
}
// byte offset of unit `u` (0..1) of row `r` inside a [rows x 16] bf16 no-swizzle tile
__device__ __forceinline__ uint32_t tail_off(int r, int u) {
  return (uint32_t)((r >> 3) * 256 + u * 128 + (r & 7) * 16);
}
// byte offset of the 16-byte unit holding columns [8u, 8u + 8) of row `r` in a tile whose 64-column chunks are
// `chunk_bytes` apart (= rows * 128) and that has MAIN such chunks before the tail
template <int MAIN>
__device__ __forceinline__ uint32_t tile_unit_off(int r, int u, uint32_t chunk_bytes) {
  return u < MAIN * 8 ? (uint32_t)(u >> 3) * chunk_bytes + sw128_off(r, u & 7)
                      : (uint32_t)MAIN * chunk_bytes + tail_off(r, u - MAIN * 8);
}
// 1-D bulk copy global -> this CTA's shared memory, completion (bytes) on an mbarrier.  size % 16 == 0.
__device__ __forceinline__ void bulk_load_1d(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
      "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
      : "memory");
}
#endif

}  // namespace osb
