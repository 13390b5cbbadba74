// HBM-bound row kernels of the denoiser block path (no tensor cores: these are bandwidth work).
//
// osb_ln_modulate: LayerNorm without affine (fp32 two-pass statistics on a register-resident row)
// fused with the adaLN modulate (1 + scale) * x + shift; one warp per row, 16-byte vector access,
// algorithmic traffic = read x + write y = 4 bytes per element.
// Replaces: opensora/models/mmdit/layers.py:205-206,223-224,248,252,312,400 and upstream v1.2
// t2i_modulate(norm(x), shift, scale) (SURVEY.md §8a-S).
//
// osb_ln_modulate_fp8 / osb_quant_rows_fp8: the FP8 (e4m3) row quantization of the opt-in MLP path, s = amax / 448 per
// row, codes e4m3_rn_satfinite(x / s); the row is register-resident, so its amax is one more warp reduction.
#include "common.cuh"

namespace osb {

constexpr int kLnWarpsPerBlock = 8;

template <int NCH>  // 16-byte chunks per lane (row has C/8 chunks, lane handles chunk lane + 32*i)
__global__ void __launch_bounds__(kLnWarpsPerBlock * 32)
ln_modulate_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ shift,
                   const float* __restrict__ scale, __nv_bfloat16* __restrict__ y, int64_t rows, int C,
                   int64_t group_rows, const int32_t* __restrict__ mod_index, int64_t mod_stride, float eps,
                   const RowScatter rsc) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kLnWarpsPerBlock + (threadIdx.x >> 5);
  pdl_wait();
  pdl_launch_dependents();
  if (row >= rows) return;
  const int nchunks = C >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);

  float v[NCH][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      uint4 t;
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                   : "=r"(t.x), "=r"(t.y), "=r"(t.z), "=r"(t.w) : "l"(xr + c));
      const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack_bf16x2(tw[e]);
        v[i][2 * e] = f.x;
        v[i][2 * e + 1] = f.y;
        sum += f.x + f.y;
      }
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[i][e] = 0.f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = v[i][e] - mean;
        sq += d * d;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / (float)C + eps);

  int64_t g = row / group_rows;
  if (mod_index) g = mod_index[g];
  const float* sh = shift + g * mod_stride;
  const float* sc = scale + g * mod_stride;
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
  if (rsc.mode != 0) {   // sequence parallel: the row goes straight into the buffer of the rank that consumes it (NVLink store)
    int peer;
    int64_t drow;
    scatter_row(rsc, row, peer, drow);
    yr = reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(scatter_base(rsc, peer)) + drow * C);
  }
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      const float4 s0 = __ldg(reinterpret_cast<const float4*>(sc + c * 8));
      const float4 s1 = __ldg(reinterpret_cast<const float4*>(sc + c * 8 + 4));
      const float4 h0 = __ldg(reinterpret_cast<const float4*>(sh + c * 8));
      const float4 h1 = __ldg(reinterpret_cast<const float4*>(sh + c * 8 + 4));
      const float s[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
      const float hh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = (v[i][e] - mean) * rstd * (1.0f + s[e]) + hh[e];
      uint4 t;
      t.x = pack_bf16x2(o[0], o[1]);
      t.y = pack_bf16x2(o[2], o[3]);
      t.z = pack_bf16x2(o[4], o[5]);
      t.w = pack_bf16x2(o[6], o[7]);
      yr[c] = t;
    }
  }
}

// ---- FP8 (e4m3) row quantization (e4m3x2: common.cuh) ---------------------------------------------------------------
// the row scale from the warp's partial amax values: amax / 448, 1 for an all-zero row
__device__ __forceinline__ float fp8_row_scale(float amax) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  return amax > 0.f ? amax / 448.0f : 1.0f;
}
// eight values -> eight codes (x / s, IEEE division as the contract states it)
__device__ __forceinline__ uint2 e4m3x8(const float (&o)[8], float s) {
  uint2 q;
  q.x = e4m3x2(o[0] / s, o[1] / s) | (e4m3x2(o[2] / s, o[3] / s) << 16);
  q.y = e4m3x2(o[4] / s, o[5] / s) | (e4m3x2(o[6] / s, o[7] / s) << 16);
  return q;
}

// osb_ln_modulate with the fp32 result quantized per row: the modulated row replaces the input row in registers, its
// amax is reduced over the warp, and the codes go out as 8 bytes per 16-byte input chunk.
template <int NCH>
__global__ void __launch_bounds__(kLnWarpsPerBlock * 32)
ln_modulate_fp8_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ shift,
                       const float* __restrict__ scale, uint8_t* __restrict__ y8, float* __restrict__ y_scale, int64_t rows,
                       int C, int64_t group_rows, const int32_t* __restrict__ mod_index, int64_t mod_stride, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kLnWarpsPerBlock + (threadIdx.x >> 5);
  pdl_wait();
  pdl_launch_dependents();
  if (row >= rows) return;
  const int nchunks = C >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);

  float v[NCH][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      uint4 t;
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                   : "=r"(t.x), "=r"(t.y), "=r"(t.z), "=r"(t.w) : "l"(xr + c));
      const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack_bf16x2(tw[e]);
        v[i][2 * e] = f.x;
        v[i][2 * e + 1] = f.y;
        sum += f.x + f.y;
      }
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[i][e] = 0.f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = v[i][e] - mean;
        sq += d * d;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / (float)C + eps);

  int64_t g = row / group_rows;
  if (mod_index) g = mod_index[g];
  const float* sh = shift + g * mod_stride;
  const float* sc = scale + g * mod_stride;
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      const float4 s0 = __ldg(reinterpret_cast<const float4*>(sc + c * 8));
      const float4 s1 = __ldg(reinterpret_cast<const float4*>(sc + c * 8 + 4));
      const float4 h0 = __ldg(reinterpret_cast<const float4*>(sh + c * 8));
      const float4 h1 = __ldg(reinterpret_cast<const float4*>(sh + c * 8 + 4));
      const float s[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
      const float hh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        v[i][e] = (v[i][e] - mean) * rstd * (1.0f + s[e]) + hh[e];
        amax = fmaxf(amax, fabsf(v[i][e]));
      }
    }
  }
  const float rs = fp8_row_scale(amax);
  if (lane == 0) y_scale[row] = rs;
  uint2* yr = reinterpret_cast<uint2*>(y8 + row * C);
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) yr[c] = e4m3x8(v[i], rs);
  }
}

// bf16 row -> e4m3 codes + fp32 scale in one read: the row is held as packed bf16 (4 registers per 8 elements) between
// its amax reduction and the conversion.
template <int NCH>
__global__ void __launch_bounds__(kLnWarpsPerBlock * 32)
quant_rows_fp8_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, uint8_t* __restrict__ y8, int64_t ldy,
                      float* __restrict__ y_scale, int64_t rows, int K) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kLnWarpsPerBlock + (threadIdx.x >> 5);
  pdl_wait();
  pdl_launch_dependents();
  if (row >= rows) return;
  const int nchunks = K >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
  uint4 t[NCH];
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                   : "=r"(t[i].x), "=r"(t[i].y), "=r"(t[i].z), "=r"(t[i].w) : "l"(xr + c));
      const uint32_t tw[4] = {t[i].x, t[i].y, t[i].z, t[i].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack_bf16x2(tw[e]);
        amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
  }
  const float rs = fp8_row_scale(amax);
  if (lane == 0) y_scale[row] = rs;
  uint2* yr = reinterpret_cast<uint2*>(y8 + row * ldy);
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      const uint32_t tw[4] = {t[i].x, t[i].y, t[i].z, t[i].w};
      float o[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack_bf16x2(tw[e]);
        o[2 * e] = f.x;
        o[2 * e + 1] = f.y;
      }
      yr[c] = e4m3x8(o, rs);
    }
  }
}

// bf16 -> e4m3 codes with one scale per (row, 128-column block): the 16 lanes of a half-warp hold one block, 8 elements
// (one 16-byte load) each, so the block amax is four shuffles and every lane stores its 8 codes.  K / 8 is a multiple of
// 16: a half-warp never straddles two blocks, and past the end whole half-warps leave together.
__global__ void __launch_bounds__(kLnWarpsPerBlock * 32)
quant_blocks_fp8_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, uint8_t* __restrict__ y8, int64_t ldy,
                        float* __restrict__ y_scale, int64_t lds, int64_t rows, int K) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t nchunks = K >> 3;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * nchunks) return;
  const int64_t row = i / nchunks;
  const int c = (int)(i - row * nchunks);
  uint4 t;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(t.x), "=r"(t.y), "=r"(t.z), "=r"(t.w) : "l"(x + row * ldx + c * 8));
  const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
  float o[8];
  float amax = 0.f;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = unpack_bf16x2(tw[e]);
    o[2 * e] = f.x;
    o[2 * e + 1] = f.y;
    amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
  }
  const unsigned half = (threadIdx.x & 16) ? 0xffff0000u : 0x0000ffffu;
#pragma unroll
  for (int m = 8; m > 0; m >>= 1) amax = fmaxf(amax, __shfl_xor_sync(half, amax, m));
  const float s = amax > 0.f ? amax / 448.0f : 1.0f;
  if ((c & 15) == 0) y_scale[row * lds + (c >> 4)] = s;
  *reinterpret_cast<uint2*>(y8 + row * ldy + c * 8) = e4m3x8(o, s);
}

// Per-row quantization of rows of any length (the MLP weights at enable time, K up to 5 x 4096): one warp per row reads
// it twice, once for the amax and once for the codes (the second read mostly hits L2).  Not on the per-step path.
__global__ void __launch_bounds__(kLnWarpsPerBlock * 32)
quant_rows_long_fp8_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, uint8_t* __restrict__ y8, int64_t ldy,
                           float* __restrict__ y_scale, int64_t lds, int64_t rows, int K) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kLnWarpsPerBlock + (threadIdx.x >> 5);
  pdl_wait();
  pdl_launch_dependents();
  if (row >= rows) return;
  const int nchunks = K >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * ldx);
  float amax = 0.f;
  for (int c = lane; c < nchunks; c += 32) {
    const uint4 t = xr[c];
    const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack_bf16x2(tw[e]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
  const float rs = fp8_row_scale(amax);
  if (lane == 0) y_scale[row * lds] = rs;
  uint2* yr = reinterpret_cast<uint2*>(y8 + row * ldy);
  for (int c = lane; c < nchunks; c += 32) {
    const uint4 t = xr[c];
    const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
    float o[8];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack_bf16x2(tw[e]);
      o[2 * e] = f.x;
      o[2 * e + 1] = f.y;
    }
    yr[c] = e4m3x8(o, rs);
  }
}

// T5LayerNorm (RMSNorm with weight): y = bf16(w * bf16(x * rsqrt(mean(x^2) + eps))), fp32 mean of squares, the two
// roundings of the reference (shardformer/modeling/t5.py:14-27, transformers T5LayerNorm).  One warp per row.
template <int NCH>
__global__ void __launch_bounds__(kLnWarpsPerBlock * 32)
rms_norm_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ y,
                int64_t rows, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * kLnWarpsPerBlock + (threadIdx.x >> 5);
  pdl_wait();
  pdl_launch_dependents();
  if (row >= rows) return;
  const int nchunks = C >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);
  float v[NCH][8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      uint4 t;
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                   : "=r"(t.x), "=r"(t.y), "=r"(t.z), "=r"(t.w) : "l"(xr + c));
      const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack_bf16x2(tw[e]);
        v[i][2 * e] = f.x;
        v[i][2 * e + 1] = f.y;
        ss += f.x * f.x + f.y * f.y;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float r = rsqrtf(ss / (float)C + eps);
  uint4* yr = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nchunks) {
      const uint4 wt = __ldg(reinterpret_cast<const uint4*>(w) + c);
      const uint32_t ww[4] = {wt.x, wt.y, wt.z, wt.w};
      uint32_t o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 wf = unpack_bf16x2(ww[e]);
        const float a = __bfloat162float(__float2bfloat16_rn(v[i][2 * e] * r));
        const float b = __bfloat162float(__float2bfloat16_rn(v[i][2 * e + 1] * r));
        o[e] = pack_bf16x2(wf.x * a, wf.y * b);
      }
      yr[c] = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

}  // namespace osb

extern "C" int osb_rms_norm(const void* x, const void* w, void* y, int64_t rows, int C, float eps, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(x && w && y, "osb_rms_norm: null tensor");
  OSB_REQUIRE(rows > 0, "osb_rms_norm: rows must be positive");
  OSB_REQUIRE(C > 0 && C % 8 == 0 && C <= 4096, "osb_rms_norm: C must be a multiple of 8 and <= 4096 (got %d)", C);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(y)) & 15) == 0,
              "osb_rms_norm: tensors must be 16-byte aligned");
  const int nch = (C / 8 + 31) / 32;
  const unsigned blocks = (unsigned)((rows + kLnWarpsPerBlock - 1) / kLnWarpsPerBlock);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* wb = static_cast<const __nv_bfloat16*>(w);
  __nv_bfloat16* yb = static_cast<__nv_bfloat16*>(y);
#define OSB_RMS_CASE(N)                                                                                       \
  if (nch <= N) {                                                                                             \
    cudaLaunchAttribute attr[2];                                                                              \
    cudaLaunchConfig_t cfg = launch_config(dim3(blocks), dim3(kLnWarpsPerBlock * 32), 0, s, attr);            \
    OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, rms_norm_kernel<N>, xb, wb, yb, rows, C, eps));                    \
    count_launch();                                                                                           \
    return OSB_OK;                                                                                            \
  }
  OSB_RMS_CASE(1) OSB_RMS_CASE(2) OSB_RMS_CASE(4) OSB_RMS_CASE(8) OSB_RMS_CASE(16)
#undef OSB_RMS_CASE
  set_error("osb_rms_norm: unsupported C %d", C);
  return OSB_ERR_UNSUPPORTED;
}

static int ln_modulate_launch(const void* x, const float* shift, const float* scale, void* y,
                              int64_t rows, int C, int64_t group_rows, const int32_t* mod_index,
                              int64_t mod_stride, float eps, const osb::RowScatter& rsc, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(x && (y || rsc.mode != 0) && shift && scale, "osb_ln_modulate: null tensor");
  OSB_REQUIRE(rows > 0, "osb_ln_modulate: rows must be positive");
  OSB_REQUIRE(C > 0 && C % 8 == 0 && C <= 8192, "osb_ln_modulate: C must be a multiple of 8 and <= 8192 (got %d)", C);
  OSB_REQUIRE(mod_stride % 4 == 0, "osb_ln_modulate: mod_stride must be a multiple of 4");
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) |
                reinterpret_cast<uintptr_t>(shift) | reinterpret_cast<uintptr_t>(scale)) & 15) == 0,
              "osb_ln_modulate: tensors must be 16-byte aligned");
  if (group_rows <= 0) group_rows = rows;
  const int nch = (C / 8 + 31) / 32;
  const unsigned blocks = (unsigned)((rows + kLnWarpsPerBlock - 1) / kLnWarpsPerBlock);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(x);
  __nv_bfloat16* yb = static_cast<__nv_bfloat16*>(y);
#define OSB_LN_CASE(N)                                                                               \
  if (nch <= N) {                                                                                    \
    cudaLaunchAttribute attr[2];                                                                     \
    cudaLaunchConfig_t cfg = launch_config(dim3(blocks), dim3(kLnWarpsPerBlock * 32), 0, s, attr);   \
    OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, ln_modulate_kernel<N>, xb, shift, scale, yb, rows, C,    \
                                      group_rows, mod_index, mod_stride, eps, rsc));                 \
    count_launch();                                                                                  \
    return OSB_OK;                                                                                   \
  }
  OSB_LN_CASE(1) OSB_LN_CASE(2) OSB_LN_CASE(3) OSB_LN_CASE(5) OSB_LN_CASE(8) OSB_LN_CASE(12)
  OSB_LN_CASE(16) OSB_LN_CASE(32)
#undef OSB_LN_CASE
  set_error("osb_ln_modulate: unsupported C %d", C);
  return OSB_ERR_UNSUPPORTED;
}

extern "C" int osb_ln_modulate(const void* x, const float* shift, const float* scale, void* y,
                               int64_t rows, int C, int64_t group_rows, const int32_t* mod_index,
                               int64_t mod_stride, float eps, void* stream) {
  return ln_modulate_launch(x, shift, scale, y, rows, C, group_rows, mod_index, mod_stride, eps, osb::RowScatter(), stream);
}

extern "C" int osb_ln_modulate_fp8(const void* x, const float* shift, const float* scale, void* y8, float* y_scale,
                                   int64_t rows, int C, int64_t group_rows, const int32_t* mod_index,
                                   int64_t mod_stride, float eps, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(x && y8 && y_scale && shift && scale, "osb_ln_modulate_fp8: null tensor");
  OSB_REQUIRE(rows > 0, "osb_ln_modulate_fp8: rows must be positive");
  // (the fp32 row stays in registers until its amax is known: beyond 4096 columns it would spill)
  OSB_REQUIRE(C > 0 && C % 8 == 0 && C <= 4096, "osb_ln_modulate_fp8: C must be a multiple of 8 and <= 4096 (got %d)", C);
  OSB_REQUIRE(mod_stride % 4 == 0, "osb_ln_modulate_fp8: mod_stride must be a multiple of 4");
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y8) |
                reinterpret_cast<uintptr_t>(shift) | reinterpret_cast<uintptr_t>(scale)) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(y_scale) & 3) == 0,
              "osb_ln_modulate_fp8: tensors must be 16-byte aligned (y_scale 4-byte)");
  if (group_rows <= 0) group_rows = rows;
  const int nch = (C / 8 + 31) / 32;
  const unsigned blocks = (unsigned)((rows + kLnWarpsPerBlock - 1) / kLnWarpsPerBlock);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(x);
  uint8_t* yb = static_cast<uint8_t*>(y8);
#define OSB_LN8_CASE(N)                                                                                  \
  if (nch <= N) {                                                                                        \
    cudaLaunchAttribute attr[2];                                                                         \
    cudaLaunchConfig_t cfg = launch_config(dim3(blocks), dim3(kLnWarpsPerBlock * 32), 0, s, attr);       \
    OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, ln_modulate_fp8_kernel<N>, xb, shift, scale, yb, y_scale, rows, \
                                      C, group_rows, mod_index, mod_stride, eps));                       \
    count_launch();                                                                                      \
    return OSB_OK;                                                                                       \
  }
  OSB_LN8_CASE(1) OSB_LN8_CASE(2) OSB_LN8_CASE(3) OSB_LN8_CASE(5) OSB_LN8_CASE(8) OSB_LN8_CASE(16)
#undef OSB_LN8_CASE
  set_error("osb_ln_modulate_fp8: unsupported C %d", C);
  return OSB_ERR_UNSUPPORTED;
}

extern "C" int osb_quant_rows_fp8(const void* x, int64_t ldx, void* y8, int64_t ldy, float* y_scale, int64_t rows, int K,
                                  void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(x && y8 && y_scale, "osb_quant_rows_fp8: null tensor");
  OSB_REQUIRE(rows > 0, "osb_quant_rows_fp8: rows must be positive");
  OSB_REQUIRE(K > 0 && K % 8 == 0 && K <= 8192, "osb_quant_rows_fp8: K must be a multiple of 8 and <= 8192 (got %d)", K);
  OSB_REQUIRE(ldx >= K && ldy >= K && ldx % 8 == 0 && ldy % 16 == 0,
              "osb_quant_rows_fp8: ldx must be a multiple of 8 and ldy of 16, both >= K (ldx %lld ldy %lld K %d)",
              (long long)ldx, (long long)ldy, K);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y8)) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(y_scale) & 3) == 0,
              "osb_quant_rows_fp8: x and y8 must be 16-byte aligned (y_scale 4-byte)");
  const int nch = (K / 8 + 31) / 32;
  const unsigned blocks = (unsigned)((rows + kLnWarpsPerBlock - 1) / kLnWarpsPerBlock);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(x);
  uint8_t* yb = static_cast<uint8_t*>(y8);
#define OSB_Q8_CASE(N)                                                                                   \
  if (nch <= N) {                                                                                        \
    cudaLaunchAttribute attr[2];                                                                         \
    cudaLaunchConfig_t cfg = launch_config(dim3(blocks), dim3(kLnWarpsPerBlock * 32), 0, s, attr);       \
    OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, quant_rows_fp8_kernel<N>, xb, ldx, yb, ldy, y_scale, rows, K)); \
    count_launch();                                                                                      \
    return OSB_OK;                                                                                       \
  }
  OSB_Q8_CASE(1) OSB_Q8_CASE(2) OSB_Q8_CASE(5) OSB_Q8_CASE(8) OSB_Q8_CASE(18) OSB_Q8_CASE(32)
#undef OSB_Q8_CASE
  set_error("osb_quant_rows_fp8: unsupported K %d", K);
  return OSB_ERR_UNSUPPORTED;
}

extern "C" int osb_quant_blocks_fp8(const void* x, int64_t ldx, void* y8, int64_t ldy, float* y_scale, int64_t lds,
                                    int64_t rows, int K, int block, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(x && y8 && y_scale, "osb_quant_blocks_fp8: null tensor");
  OSB_REQUIRE(rows > 0, "osb_quant_blocks_fp8: rows must be positive");
  OSB_REQUIRE(K > 0 && K % 128 == 0, "osb_quant_blocks_fp8: K must be a positive multiple of 128 (got %d)", K);
  OSB_REQUIRE(block == 128 || block == K, "osb_quant_blocks_fp8: block must be 128 or K (got %d, K %d)", block, K);
  OSB_REQUIRE(ldx >= K && ldy >= K && ldx % 8 == 0 && ldy % 8 == 0 && lds >= K / block,
              "osb_quant_blocks_fp8: ldx and ldy must be >= K and multiples of 8, lds >= K / block (ldx %lld ldy %lld "
              "lds %lld K %d)", (long long)ldx, (long long)ldy, (long long)lds, K);
  OSB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y8) & 7) == 0 &&
              (reinterpret_cast<uintptr_t>(y_scale) & 3) == 0,
              "osb_quant_blocks_fp8: x must be 16-byte, y8 8-byte and y_scale 4-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* xb = static_cast<const __nv_bfloat16*>(x);
  uint8_t* yb = static_cast<uint8_t*>(y8);
  cudaLaunchAttribute attr[2];
  if (block == 128) {
    const int64_t threads = rows * (K / 8);
    const int64_t blocks = (threads + kLnWarpsPerBlock * 32 - 1) / (kLnWarpsPerBlock * 32);
    OSB_REQUIRE(blocks < (1ll << 31), "osb_quant_blocks_fp8: too many rows (%lld)", (long long)rows);
    cudaLaunchConfig_t cfg = launch_config(dim3((unsigned)blocks), dim3(kLnWarpsPerBlock * 32), 0, s, attr);
    OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, quant_blocks_fp8_kernel, xb, ldx, yb, ldy, y_scale, lds, rows, K));
  } else {
    const unsigned blocks = (unsigned)((rows + kLnWarpsPerBlock - 1) / kLnWarpsPerBlock);
    cudaLaunchConfig_t cfg = launch_config(dim3(blocks), dim3(kLnWarpsPerBlock * 32), 0, s, attr);
    OSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, quant_rows_long_fp8_kernel, xb, ldx, yb, ldy, y_scale, lds, rows, K));
  }
  count_launch();
  return OSB_OK;
}

extern "C" int osb_ln_modulate_scatter(const void* x, const float* shift, const float* scale, int64_t rows, int C,
                                       int64_t group_rows, const int32_t* mod_index, int64_t mod_stride, float eps,
                                       const osb_scatter* scatter, void* stream) {
  using namespace osb;
  OSB_REQUIRE(scatter != nullptr && scatter->mode != 0, "osb_ln_modulate_scatter: no scatter given");
  RowScatter rsc;
  const int rc = make_row_scatter(&rsc, scatter, rows, "osb_ln_modulate_scatter");
  if (rc) return rc;
  return ln_modulate_launch(x, shift, scale, nullptr, rows, C, group_rows, mod_index, mod_stride, eps, rsc, stream);
}

// ------------------------------------------------------------------------------------------------------------
// osb_comm_barrier: orders the producers and consumers of a peer-memory exchange across the ranks of one NVSwitch
// domain.  One CTA; thread p < P: release-store the new epoch into slot `rank` of rank p's flag array, then spin
// (acquire loads, bounded) until slot p of the local array has reached it.  The epoch counter lives in device memory
// and is advanced by the kernel itself, so a captured CUDA graph replays correctly.
// Replaces the synchronisation half of dist.all_to_all (opensora/acceleration/communications.py:8-18).
// ------------------------------------------------------------------------------------------------------------
namespace osb {
struct BarrierParams {
  int32_t P, rank;
  uint32_t* epoch;
  uint32_t* flags_local;
  uint32_t* flags_peer[OSB_MAX_PEERS];
};
__global__ void __launch_bounds__(32) comm_barrier_kernel(const BarrierParams b) {
  const int p = threadIdx.x;
  const uint32_t e = *b.epoch + 1u;
  if (p < b.P) {
    uint32_t* dst = b.flags_peer[0];
#pragma unroll
    for (int k = 1; k < OSB_MAX_PEERS; ++k) dst = (p == k) ? b.flags_peer[k] : dst;
    // everything this rank's earlier kernels stored to peer memory is ordered before the flag (system scope)
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(dst + b.rank), "r"(e) : "memory");
    uint32_t spins = 0;
    for (;;) {
      uint32_t v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(b.flags_local + p) : "memory");
      if ((int32_t)(v - e) >= 0) break;
      if (++spins > (1u << 27)) {
        printf("osb200: comm barrier timed out (rank %d waiting for rank %d, epoch %u, saw %u)\n", b.rank, p, e, v);
        __trap();
      }
    }
  }
  __syncwarp();
  if (p == 0) *b.epoch = e;
}
}  // namespace osb

extern "C" int osb_comm_barrier(const osb_comm_barrier_args* a, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(a != nullptr && a->P >= 1 && a->P <= OSB_MAX_PEERS && a->rank >= 0 && a->rank < a->P, "osb_comm_barrier: bad ranks");
  OSB_REQUIRE(a->epoch && a->flags_local, "osb_comm_barrier: null epoch / flags");
  BarrierParams b = {};
  b.P = a->P; b.rank = a->rank; b.epoch = a->epoch; b.flags_local = a->flags_local;
  for (int p = 0; p < a->P; ++p) {
    OSB_REQUIRE(a->flags_peer[p] != nullptr, "osb_comm_barrier: null peer flag array %d", p);
    b.flags_peer[p] = a->flags_peer[p];
  }
  comm_barrier_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(b);
  OSB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return OSB_OK;
}

// ------------------------------------------------------------------------------------------------------------
// osb_cfg_euler: classifier-free-guidance combine + Euler step of the rectified-flow sampler in ONE pass:
//   pred = uncond2 + g_img * (uncond - uncond2) + g_txt * (cond - uncond)      (uncond2 == NULL: uncond + g_txt * (cond - uncond))
//   out  = x + dt * pred
// bf16 in/out, fp32 math, one rounding (the reference rounds after each of the ~7 torch ops).  g_img may be a
// per-element bf16 map (temporal oscillation, sampling.py:208-217) that repeats with period `map_period`.
// Replaces opensora/utils/sampling.py:204-222 (I2VDenoiser.denoise update).  HBM bound: 5 tensors x 2 B/element.
// ------------------------------------------------------------------------------------------------------------
namespace osb {
// The combine + Euler arithmetic of one element, shared by osb_cfg_euler and osb_rf_masked_step so that the two produce
// bit-identical latents for the same inputs (the same fp32 expression, contracted the same way).
__device__ __forceinline__ float cfg_euler_elem(float c, float u, float u2, float gi, float g_txt, float x, float dt) {
  const float p = u2 + gi * (u - u2) + g_txt * (c - u);
  return x + dt * p;
}

__global__ void __launch_bounds__(256)
cfg_euler_kernel(const uint4* __restrict__ c, const uint4* __restrict__ u, const uint4* __restrict__ u2,
                 const uint4* __restrict__ x, uint4* __restrict__ out, int64_t nvec, float g_txt, float g_img,
                 const uint4* __restrict__ g_map, int64_t map_vecs, float dt) {
  pdl_wait();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    const uint4 cv = c[i], uv = u[i], xv = x[i];
    const uint4 u2v = u2 ? u2[i] : uv;
    const uint4 gv = g_map ? g_map[i % map_vecs] : make_uint4(0, 0, 0, 0);
    const uint32_t cw[4] = {cv.x, cv.y, cv.z, cv.w}, uw[4] = {uv.x, uv.y, uv.z, uv.w}, vw[4] = {u2v.x, u2v.y, u2v.z, u2v.w};
    const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w}, gw[4] = {gv.x, gv.y, gv.z, gv.w};
    uint32_t ow[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 cf = unpack_bf16x2(cw[e]), uf = unpack_bf16x2(uw[e]), vf = unpack_bf16x2(vw[e]), xf = unpack_bf16x2(xw[e]);
      float2 gi = make_float2(g_img, g_img);
      if (g_map) gi = unpack_bf16x2(gw[e]);
      ow[e] = pack_bf16x2(cfg_euler_elem(cf.x, uf.x, vf.x, gi.x, g_txt, xf.x, dt),
                          cfg_euler_elem(cf.y, uf.y, vf.y, gi.y, g_txt, xf.y, dt));
    }
    out[i] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
  }
}
}  // namespace osb

extern "C" int osb_cfg_euler(const void* cond, const void* uncond, const void* uncond2, const void* x, void* out, int64_t n,
                             float g_txt, float g_img, const void* g_img_map, int64_t map_period, float dt, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(cond && uncond && x && out, "osb_cfg_euler: null tensor");
  OSB_REQUIRE(n > 0 && n % 8 == 0, "osb_cfg_euler: element count must be a positive multiple of 8");
  OSB_REQUIRE(g_img_map == nullptr || (map_period > 0 && map_period % 8 == 0 && n % map_period == 0),
              "osb_cfg_euler: guidance map period must be a multiple of 8 dividing n");
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(cond) | reinterpret_cast<uintptr_t>(uncond) | reinterpret_cast<uintptr_t>(uncond2) |
                reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(g_img_map)) & 15) == 0,
              "osb_cfg_euler: tensors must be 16-byte aligned");
  const int64_t nvec = n / 8;
  int64_t blocks = (nvec + 255) / 256;
  if (blocks > (int64_t)sm_count() * 16) blocks = (int64_t)sm_count() * 16;
  cfg_euler_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(cond), static_cast<const uint4*>(uncond), static_cast<const uint4*>(uncond2),
      static_cast<const uint4*>(x), static_cast<uint4*>(out), nvec, g_txt, g_img, static_cast<const uint4*>(g_img_map),
      g_img_map ? map_period / 8 : 1, dt);
  OSB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return OSB_OK;
}

// ------------------------------------------------------------------------------------------------------------
// osb_rf_masked_step: the frame-masked rectified-flow step of image / video conditioning (Open-Sora v1.2 RFLOW.sample,
// mask branch) in ONE pass over the latent: the end of step i (combine + Euler update of the frames being generated)
// fused with the start of step i + 1 (re-noising of the frames whose edit ratio the schedule has just reached).
// Per frame (b, f), with m = frame_mask[b, f] * N:
//   upd     = update && m >= t_cur[b]                     z' = upd ? z + dt * (vu + g (vc - vu)) : z   (dt = (t_cur - t_next) * (1/N))
//   prev    = update ? upd : frame_mask[b, f] == 1
//   renoise = noise && m >= t_next[b] && !prev            out = renoise ? (1 - a) z' + a noise : z'    (a = t_next * (1/N))
// A frame is never both updated and re-noised in one pass, so every output element is rounded once.  Frames left alone
// are copied bit for bit (in place: not written at all).  HBM bound: up to 5 tensors x 2 B/element.
// ------------------------------------------------------------------------------------------------------------
namespace osb {
struct MaskedFrame {
  bool upd, renoise;
  float dt, a;
};

__device__ __forceinline__ MaskedFrame masked_frame(int64_t row, int T, int64_t CT, const float* __restrict__ fm,
                                                    const float* __restrict__ tc, const float* __restrict__ tn, float N,
                                                    bool update, bool has_noise) {
  const int64_t b = row / CT;
  const float mv = __ldg(fm + b * T + row % T);
  const float m = mv * N;
  const float t0 = __ldg(tc + b), t1 = __ldg(tn + b);
  MaskedFrame r;
  r.upd = update && m >= t0;
  const bool prev = update ? r.upd : mv == 1.0f;
  r.renoise = has_noise && m >= t1 && !prev;
  r.dt = (t0 - t1) * (1.0f / N);   // torch's (t_cur - t_next) / N on the GPU: the t2v loop's dt, to the bit
  r.a = t1 * (1.0f / N);
  return r;
}

__device__ __forceinline__ float renoise_elem(float x, float n, float a) { return (1.0f - a) * x + a * n; }

// kVec: 8 elements (one uint4) per unit, H*W % 8 == 0 so a unit never straddles two frames; else one element per unit
template <bool kVec>
__global__ void __launch_bounds__(256)
rf_masked_step_kernel(const __nv_bfloat16* __restrict__ c, const __nv_bfloat16* __restrict__ u, const __nv_bfloat16* x,
                      const __nv_bfloat16* __restrict__ noise, __nv_bfloat16* out, const float* __restrict__ fm,
                      const float* __restrict__ tc, const float* __restrict__ tn, int64_t units, int64_t units_per_row,
                      int T, int64_t CT, float g, float N, int update) {
  pdl_wait();
  const bool in_place = out == x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < units; i += (int64_t)gridDim.x * blockDim.x) {
    const MaskedFrame f = masked_frame(i / units_per_row, T, CT, fm, tc, tn, N, update != 0, noise != nullptr);
    if (in_place && !f.upd && !f.renoise) continue;
    if constexpr (kVec) {
      const uint4 xv = reinterpret_cast<const uint4*>(x)[i];
      uint4 ov = xv;
      const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
      uint32_t ow[4];
      if (f.upd) {
        const uint4 cv = reinterpret_cast<const uint4*>(c)[i], uv = reinterpret_cast<const uint4*>(u)[i];
        const uint32_t cw[4] = {cv.x, cv.y, cv.z, cv.w}, uw[4] = {uv.x, uv.y, uv.z, uv.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 cf = unpack_bf16x2(cw[e]), uf = unpack_bf16x2(uw[e]), xf = unpack_bf16x2(xw[e]);
          ow[e] = pack_bf16x2(cfg_euler_elem(cf.x, uf.x, uf.x, 1.0f, g, xf.x, f.dt),
                              cfg_euler_elem(cf.y, uf.y, uf.y, 1.0f, g, xf.y, f.dt));
        }
        ov = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      } else if (f.renoise) {
        const uint4 nv = reinterpret_cast<const uint4*>(noise)[i];
        const uint32_t nw[4] = {nv.x, nv.y, nv.z, nv.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 nf = unpack_bf16x2(nw[e]), xf = unpack_bf16x2(xw[e]);
          ow[e] = pack_bf16x2(renoise_elem(xf.x, nf.x, f.a), renoise_elem(xf.y, nf.y, f.a));
        }
        ov = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      }
      reinterpret_cast<uint4*>(out)[i] = ov;
    } else {
      __nv_bfloat16 o = x[i];
      if (f.upd) {
        const float uf = __bfloat162float(u[i]);
        o = __float2bfloat16_rn(cfg_euler_elem(__bfloat162float(c[i]), uf, uf, 1.0f, g, __bfloat162float(o), f.dt));
      } else if (f.renoise) {
        o = __float2bfloat16_rn(renoise_elem(__bfloat162float(o), __bfloat162float(noise[i]), f.a));
      }
      out[i] = o;
    }
  }
}
}  // namespace osb

extern "C" int osb_rf_masked_step(const void* cond, const void* uncond, const void* x, const void* noise, void* out,
                                  const float* frame_mask, const float* t_cur, const float* t_next, int32_t B, int32_t C,
                                  int32_t T, int64_t HW, float guidance, int32_t num_timesteps, int32_t update, void* stream) {
  using namespace osb;
  if (!initialised()) { set_error("osb_init() has not been called"); return OSB_ERR_NOT_INIT; }
  OSB_REQUIRE(x && out && frame_mask && t_cur && t_next, "osb_rf_masked_step: null tensor");
  OSB_REQUIRE(!update || (cond && uncond), "osb_rf_masked_step: the update needs cond and uncond");
  OSB_REQUIRE(update || noise, "osb_rf_masked_step: without the update there must be noise to add");
  OSB_REQUIRE(B > 0 && C > 0 && T > 0 && HW > 0, "osb_rf_masked_step: B, C, T, H*W must be positive");
  OSB_REQUIRE(num_timesteps > 0, "osb_rf_masked_step: num_timesteps must be positive");
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(cond) | reinterpret_cast<uintptr_t>(uncond) | reinterpret_cast<uintptr_t>(x) |
                reinterpret_cast<uintptr_t>(noise) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
              "osb_rf_masked_step: bf16 tensors must be 16-byte aligned");
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(frame_mask) | reinterpret_cast<uintptr_t>(t_cur) |
                reinterpret_cast<uintptr_t>(t_next)) & 3) == 0,
              "osb_rf_masked_step: fp32 tensors must be 4-byte aligned");
  const bool vec = HW % 8 == 0;
  const int64_t CT = (int64_t)C * T;
  const int64_t units_per_row = vec ? HW / 8 : HW;
  const int64_t units = (int64_t)B * CT * units_per_row;
  int64_t blocks = (units + 255) / 256;
  if (blocks > (int64_t)sm_count() * 16) blocks = (int64_t)sm_count() * 16;
  const auto* cb = static_cast<const __nv_bfloat16*>(cond);
  const auto* ub = static_cast<const __nv_bfloat16*>(uncond);
  const auto* xb = static_cast<const __nv_bfloat16*>(x);
  const auto* nb = static_cast<const __nv_bfloat16*>(noise);
  auto* ob = static_cast<__nv_bfloat16*>(out);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (vec)
    rf_masked_step_kernel<true><<<(unsigned)blocks, 256, 0, s>>>(cb, ub, xb, nb, ob, frame_mask, t_cur, t_next, units,
                                                                 units_per_row, T, CT, guidance, (float)num_timesteps, update);
  else
    rf_masked_step_kernel<false><<<(unsigned)blocks, 256, 0, s>>>(cb, ub, xb, nb, ob, frame_mask, t_cur, t_next, units,
                                                                  units_per_row, T, CT, guidance, (float)num_timesteps, update);
  OSB_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return OSB_OK;
}
