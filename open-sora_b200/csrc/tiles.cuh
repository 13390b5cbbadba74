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
// The same bytes serve as the operand of S = Q K^T and of O = P V: as wgmma shared-memory descriptors (the chunks
// K-major / MN-major with the 128-byte swizzle, the tail as no-swizzle core matrices) or through ldmatrix / .trans.
// Producers: the head-tile epilogue of gemm_bf16_kernel (bias + per-head RMSNorm + RoPE fused, gemm_sm90.cu) and the
// staging step of attn_short_kernel.  Consumers: attn_tiles_kernel (wgmma), attn_short_kernel (ldmatrix + mma.sync),
// both in attn_sm90.cu, and head_tiles_fp8_kernel (attn_fp8_sm90.cu).
//
// FP8 head tiles (osb_head_tiles_fp8 -> osb_attn_tiles_fp8, attn_fp8_sm90.cu): every bf16 tile has an e4m3 twin
// of 128 rows x 128 bytes (kTileF8Bytes), again the shared-memory image of a wgmma operand: K-major rows of 128 bytes
// in the 128-byte swizzle (byte c of row r at r * 128 + (((c / 16) ^ (r % 8)) * 16) + c % 16), loaded by one bulk copy.
//   q / k tile: row = tile row (token), byte = channel; channels >= D and rows >= tile_rows hold zero codes.  The head
//               dim is padded to 128 bytes but the QK^T product runs ceil(D / 32) k32 steps only (3 for D = 72).
//   v tile:     row = channel (< D; later rows unused), byte p = key vt8_key(p) of the tile (below), so the
//               S accumulator registers are the A fragment of the PV product as they are.
// Next to the codes, 128 fp32 scales per tile (kTileF8Scales): per row for q / k (1 past the tile's rows), per
// channel for v (1 for channels >= D).  Tile (kind, head, t) has index (kind * heads + head) * tiles_per_head + t in
// both arrays, the indexing of the bf16 buffer it was converted from.
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

constexpr int kTileF8Bytes = 128 * 128;
constexpr int kTileF8Scales = 128;

// How GEMM rows (tokens) map to (tile, row in tile); shared by the producing epilogue and by the attention kernel's
// output addressing (the inverse map).
//   mode 0: sequences are contiguous row blocks: seq = row / L, pos = row % L                (spatial, cross, text)
//   mode 1: frame-major token stream viewed along T: row = (b*T + t)*S + s -> seq = b*S + s, pos = t    (temporal)
//   G > 1 : G short sequences packed per tile: tile = seq / G, r = (seq % G) * L + pos              (G * L <= TR)
//   G == 1: tile = seq * tps + pos / TR, r = pos % TR                                       (tps = ceil(L / TR))
struct TileMap {
  int32_t mode, L, S, T, G, tps, TR;
};

// 32-bit arithmetic: the host requires fewer than 2^31 token rows
__host__ __device__ __forceinline__ void tile_of_row(const TileMap& m, uint32_t row, uint32_t& tile, uint32_t& pos, int& r) {
  uint32_t seq;
  if (m.mode == 0) {
    seq = row / (uint32_t)m.L;
    pos = row - seq * (uint32_t)m.L;
  } else {
    const uint32_t ts = (uint32_t)m.T * (uint32_t)m.S;
    const uint32_t b = row / ts;
    const uint32_t rem = row - b * ts;
    pos = rem / (uint32_t)m.S;
    seq = b * (uint32_t)m.S + (rem - pos * (uint32_t)m.S);
  }
  if (m.G > 1) {
    tile = seq / (uint32_t)m.G;
    r = (int)((seq - tile * (uint32_t)m.G) * (uint32_t)m.L + pos);
  } else {
    const uint32_t jt = pos / (uint32_t)m.TR;
    tile = seq * (uint32_t)m.tps + jt;
    r = (int)(pos - jt * (uint32_t)m.TR);
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
// position p (0..31) of a 32-key group of vt8 holds key j(p) = 16 (p/16) + 2 ((p%16)/4) + p%2 + 8 ((p%4)/2): the order in
// which a thread's S accumulator registers (columns 2 (lane%4) + {0, 1, 8, 9, 16, 17, 24, 25}) fill its FP8 A fragment
// (k = 4 (lane%4) + {0..3, 16..19})
__device__ __forceinline__ int vt8_key(int pos) {
  return (pos & ~31) + 16 * ((pos >> 4) & 1) + 2 * ((pos >> 2) & 3) + (pos & 1) + 8 * ((pos >> 1) & 1);
}
// 1-D bulk copy global -> this CTA's shared memory, completion (bytes) on an mbarrier.  size % 16 == 0.
__device__ __forceinline__ void bulk_load_1d(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
      "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
      : "memory");
}

// Key sets and output rows of the head-tile attention kernels (osb_attn_tiles, osb_attn_tiles_fp8).  Key set i belongs
// to sequence i (G == 1: qmap.tps query tiles, nkb key tiles, Lk key slots clipped by kv_lens) or to query tile i
// (G > 1: one key tile, the keys of its sequence g in the slots [g Lk, g Lk + Lk)).
struct TileSets {
  TileMap qmap;             // q tiles <-> rows of `out`
  int32_t BK, nkb, Lk;      // key-tile rows, key tiles per set, keys per sequence
  int64_t num_seqs, num_sets;
  const int32_t* kv_lens;
  __nv_bfloat16* out;
  int64_t out_ld;
  RowScatter out_sc;        // sequence parallel: output rows go straight to the consuming rank's buffer
};

// valid key slots of a set: packed tiles G * Lk, else Lk clipped by kv_lens
__device__ __forceinline__ int tile_set_keys(const TileSets& t, int64_t set) {
  int keys = t.qmap.G > 1 ? t.qmap.G * t.Lk : t.Lk;
  if (t.qmap.G == 1 && t.kv_lens) { const int l = __ldg(t.kv_lens + set); keys = l < keys ? (l < 0 ? 0 : l) : keys; }
  return keys;
}

// row r of query tile qt of `set` (keys = tile_set_keys(t, set)): its sequence and position, whether it holds a token,
// and the key slots [lo, hi) it attends to (empty when it holds none)
__device__ __forceinline__ void tile_query_row(const TileSets& t, int64_t set, int qt, int keys, int r, int64_t& seq,
                                               int& pos, bool& valid, int& lo, int& hi) {
  lo = hi = 0;
  if (t.qmap.G > 1) {
    const int g = r / t.qmap.L;
    pos = r - g * t.qmap.L;
    seq = set * t.qmap.G + g;
    valid = g < t.qmap.G && seq < t.num_seqs;
    if (valid) { lo = g * t.Lk; hi = lo + t.Lk; }
  } else {
    pos = qt * t.qmap.TR + r;
    seq = set;
    valid = r < t.qmap.TR && pos < t.qmap.L;
    if (valid) hi = keys;
  }
}

// first element of the output row of token `pos` of sequence `seq`: the inverse q map, then the optional scatter
__device__ __forceinline__ __nv_bfloat16* tile_out_row(const TileSets& t, int64_t seq, int pos) {
  int64_t orow = row_of_token(t.qmap, seq, pos);
  __nv_bfloat16* obase = t.out;
  if (t.out_sc.mode != 0) {
    int peer;
    scatter_row(t.out_sc, orow, peer, orow);
    obase = static_cast<__nv_bfloat16*>(scatter_base(t.out_sc, peer));
  }
  return obase + orow * t.out_ld;
}

// Host checks shared by the entry points (attn_sm90.cu).  `who` names the entry point in the error message.
// osb_tile_map -> TileMap
int make_tile_map(TileMap* dst, const osb_tile_map& m, const char* who);
// the key-set and output fields of osb_attn_tiles_args -> TileSets
int make_tile_sets(TileSets* dst, const osb_attn_tiles_args* a, const char* who);
#endif

}  // namespace osb
