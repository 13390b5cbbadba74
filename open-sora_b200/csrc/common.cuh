// Shared device/host helpers for the osb200 sm_90a kernels: mbarrier, TMA, wgmma and mma.sync PTX
// wrappers, error plumbing for the C ABI.  Hand-written for Hopper (sm_90a).
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/osb200.h"

namespace osb {

// ------------------------------------------------------------------------------------------
// host side: error handling and launch accounting
// ------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);
bool initialised();
int sm_count();

#define OSB_CHECK_CUDA(expr)                                                            \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      osb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,  \
                     __LINE__);                                                         \
      return OSB_ERR_CUDA;                                                              \
    }                                                                                   \
  } while (0)

#define OSB_REQUIRE(cond, ...)              \
  do {                                      \
    if (!(cond)) {                          \
      osb::set_error(__VA_ARGS__);          \
      return OSB_ERR_INVALID;               \
    }                                       \
  } while (0)

// Encode a 2D tiled tensor map over a row-major bf16 matrix [rows, cols] with row stride `ld`
// elements; box = box_rows x box_cols, 128-byte swizzle (box_cols must be 64), zero OOB fill.
// Launch configuration shared by every kernel: grid / block / smem / stream + the PDL attribute (and an optional
// cluster dimension).  `attrs` must have room for 2 entries and outlive the launch call.
bool pdl_enabled();
inline cudaLaunchConfig_t launch_config(dim3 grid, dim3 block, size_t smem, cudaStream_t stream, cudaLaunchAttribute* attrs,
                                        unsigned cluster_x = 1) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  unsigned n = 0;
  if (cluster_x > 1) {
    attrs[n].id = cudaLaunchAttributeClusterDimension;
    attrs[n].val.clusterDim.x = cluster_x;
    attrs[n].val.clusterDim.y = 1;
    attrs[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl_enabled()) {
    attrs[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attrs;
  cfg.numAttrs = n;
  return cfg;
}

int make_tmap_2d_bf16(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t ld, uint32_t box_rows, uint32_t box_cols);
// the same over a one-byte e4m3 matrix (box_cols must be 128: one 128-byte swizzle row)
int make_tmap_2d_e4m3(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t ld, uint32_t box_rows, uint32_t box_cols);

// `batch` such bf16 matrices `batch_ld` ELEMENTS apart as a 3D map (column, row, sample): rows past `rows` of a sample
// are zero filled, never the next sample's.  Box = box_rows x 64 columns of one sample, 128-byte swizzle.
int make_tmap_3d_bf16(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint64_t batch,
                      uint64_t batch_ld, uint32_t box_rows, uint32_t box_cols);

struct RowScatter;
// validates an osb_scatter and copies it into the kernel-parameter form; rows = rows the producer writes
int make_row_scatter(RowScatter* dst, const osb_scatter* src, int64_t rows, const char* who);

// 5D tiled tensor map over bf16 data: dims/box/element strides innermost first, strides in BYTES for
// dims 1..4 (multiples of 16), 128-byte swizzle (box[0] must be 64 elements), zero OOB fill.
int make_tmap_5d_bf16(CUtensorMap* map, const void* base, const uint64_t dims[5], const uint64_t strides_bytes[4],
                      const uint32_t box[5], const uint32_t elem_strides[5]);

// ------------------------------------------------------------------------------------------
// device side
// ------------------------------------------------------------------------------------------
#ifdef __CUDACC__

#ifndef OSB_SPIN_LIMIT
#define OSB_SPIN_LIMIT (1u << 24)  // bounded waits: a protocol bug traps instead of hanging the box
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive on the barrier at the same smem offset in CTA `cta` of this cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}\n" ::"r"(bar),
      "r"(cta)
      : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe (try_wait may park the thread for a system-dependent time before reporting failure)
__device__ __forceinline__ bool mbar_test_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\tmbarrier.test_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > OSB_SPIN_LIMIT) {
      printf("osb200: mbarrier wait timed out (block %d thread %d bar 0x%x parity %u)\n",
             blockIdx.x, threadIdx.x, bar, parity);
      __trap();
    }
  }
}
// the same bounded wait with no call on its timeout path: inside a wgmma region a function call (printf) makes ptxas
// serialise every wgmma.mma_async of the kernel (C7510), so wgmma consumers wait with this one
__device__ __forceinline__ void mbar_wait_notrace(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > OSB_SPIN_LIMIT) __trap();
  }
}
// acquire at cluster scope (used when the arrivals come from the peer CTA)
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) break;
    if (++spins > OSB_SPIN_LIMIT) {
      printf("osb200: cluster mbarrier wait timed out (block %d thread %d)\n", blockIdx.x,
             threadIdx.x);
      __trap();
    }
  }
}

// ---- cluster -----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;"
               ::: "memory");
}

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------
// Every osb200 kernel is launched with cudaLaunchAttributeProgrammaticStreamSerialization (osb::launch_config):
// its prologue (barrier init, descriptor prefetch) may overlap the tail of the previous kernel in
// the stream; pdl_wait() must precede the first access to memory the previous kernel may have written, and
// pdl_launch_dependents() lets the next kernel's CTAs start filling SMs this kernel has already vacated.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- proxy fences ------------------------------------------------------------------------
// make generic-proxy smem writes visible to the async proxy (TMA / tensor core operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA ---------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2D tile load into this CTA's smem, completion on this CTA's mbarrier
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint32_t bar, uint32_t dst,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// 3D tile load (a [rows, ld] matrix per sample: coordinates column, row, sample)
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint32_t bar, uint32_t dst, int32_t c0, int32_t c1,
                                            int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// 5D tile loads (NDHWC activations of the causal-conv VAE: coordinates c, w, h, t, n)
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* m, uint32_t bar, uint32_t dst, int32_t c0,
                                            int32_t c1, int32_t c2, int32_t c3, int32_t c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// tile stores from this CTA's smem (box elements outside the tensor map's extents are not written); the smem writes they
// read must be made visible to the async proxy first (fence_proxy_async_smem + a barrier over the writing threads)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, uint32_t src, int32_t c0, int32_t c1, int32_t c2,
                                             int32_t c3, int32_t c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed bulk store has finished READING its smem source (the smem may be reused or released)
__device__ __forceinline__ void bulk_wait_group_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// named barrier `id` (1..15) over `count` threads (a multiple of 32)
__device__ __forceinline__ void named_barrier_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
// ---- wgmma (warpgroup MMA) ----------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// shared-memory matrix descriptor (sm_90), K-major operand, 128-byte swizzle, rows of 64 bf16 (128 B),
// 8-row swizzle atoms 1024 B apart.  The tile base must be 1024-byte aligned; +32 B along K = +2.
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);        // start address  [0,14)
  d |= static_cast<uint64_t>(1) << 16;                            // LBO (unused for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                    // SBO = 1024 B   [32,46)
  d |= static_cast<uint64_t>(1) << 62;                            // SWIZZLE_128B
  return d;
}

// ---- mma.sync / ldmatrix (register-operand tensor core path of the attention kernels) -----------------
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
// D[16 x 8] += A[16 x 16] * B[16 x 8], bf16 operands, fp32 accumulator
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---- output row routing to peer buffers (osb_scatter) ----------------------------------------------------------
struct RowScatter {
  int32_t mode, P, rank, I, J;
  void* peer[OSB_MAX_PEERS];
};
__device__ __forceinline__ void scatter_row(const RowScatter& sc, int64_t row, int& peer, int64_t& dst_row) {
  const uint32_t ij = (uint32_t)sc.I * (uint32_t)sc.J;
  const uint32_t b = (uint32_t)(row / ij);
  const uint32_t rem = (uint32_t)(row - (int64_t)b * ij);
  const uint32_t i = rem / (uint32_t)sc.J, j = rem - i * (uint32_t)sc.J;
  if (sc.mode == 1) {
    const uint32_t jc = (uint32_t)sc.J / (uint32_t)sc.P;
    const uint32_t p = j / jc;
    peer = (int)p;
    dst_row = ((int64_t)b * sc.P * sc.I + (int64_t)sc.rank * sc.I + i) * jc + (j - p * jc);
  } else if (sc.mode == 3) {          // transpose in place of the rank: [B, I, J] -> [B, J, I]
    peer = sc.rank;
    dst_row = ((int64_t)b * sc.J + j) * sc.I + i;
  } else if (sc.mode == 4) {          // split J like mode 1, destination transposed: rank p holds [B, J/P, P*I]
    const uint32_t jc = (uint32_t)sc.J / (uint32_t)sc.P;
    const uint32_t p = j / jc;
    peer = (int)p;
    dst_row = ((int64_t)b * jc + (j - p * jc)) * ((int64_t)sc.P * sc.I) + (int64_t)sc.rank * sc.I + i;
  } else {
    const uint32_t ic = (uint32_t)sc.I / (uint32_t)sc.P;
    const uint32_t p = i / ic;
    peer = (int)p;
    dst_row = ((int64_t)b * ic + (i - p * ic)) * ((int64_t)sc.P * sc.J) + (int64_t)sc.rank * sc.J + j;
  }
}
// peer[] selected without a runtime index into the parameter struct (which would move it to local memory)
__device__ __forceinline__ void* scatter_base(const RowScatter& sc, int peer) {
  void* b = sc.peer[0];
#pragma unroll
  for (int k = 1; k < OSB_MAX_PEERS; ++k) b = (peer == k) ? sc.peer[k] : b;
  return b;
}

// ---- small math helpers ------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
// 2^x as ONE MUFU op (exp2f() adds a denormal-range fix-up: 3 extra instructions per element in softmax loops);
// results below 2^-126 flush to zero, which is what a softmax weight that small should be.
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// GELU, tanh approximation (torch.nn.GELU(approximate="tanh"); layers.py:279).  tanh.approx.f32 is one
// MUFU op with ~2^-11 relative error - an order of magnitude below the bf16 rounding of the result.
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * (x + k1 * x * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * (1.0f + t);
}

// two e4m3 codes, round to nearest even, saturated to +-448 (`lo` in the low byte)
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

#endif  // __CUDACC__
}  // namespace osb
