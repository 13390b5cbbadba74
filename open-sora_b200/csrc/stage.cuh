// Staging math of one attention head row, shared by the bf16 attention kernels (attn_sm90.cu, which store the row into
// a shared-memory tile) and the FP8 attention prep (attn_fp8_sm90.cu, which quantizes it): optional per-head RMSNorm
// with weight, optional RoPE in either layout, in fp32, one rounding to bf16.
#pragma once

#include "common.cuh"

namespace osb {

// Checks of osb_attn_short_args shared by osb_attn_short and osb_attn_fp8 (attn_sm90.cu): null and empty problems, the
// norm-weight and RoPE pairs, leading dimensions and alignment.  `who` names the entry point in the error message.
int check_attn_short_args(const osb_attn_short_args* a, const char* who);

#ifdef __CUDACC__
__device__ __forceinline__ void unpack8(const uint4& t, float* x) {
  const uint32_t tw[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = unpack_bf16x2(tw[e]);
    x[2 * e] = f.x;
    x[2 * e + 1] = f.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float* x) {
  uint4 o;
  o.x = pack_bf16x2(x[0], x[1]);
  o.y = pack_bf16x2(x[2], x[3]);
  o.z = pack_bf16x2(x[4], x[5]);
  o.w = pack_bf16x2(x[6], x[7]);
  return o;
}

// One head row of U raw bf16x8 units, in place: optional RMSNorm scale r*w and RoPE in fp32 -> bf16.  Works unit by
// unit (a rotate-half pair of units at a time) so that no fp32 copy of the whole row is live.
template <int D, int U>
__device__ __forceinline__ void norm_rope_row(uint4 (&raw)[U], bool norm, float eps, const __nv_bfloat16* w,
                                              const float* cosr, const float* sinr, bool rope_half) {
  float r = 1.f;
  if (norm) {
    float ss = 0.f;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float x[8];
      unpack8(raw[u], x);
#pragma unroll
      for (int e = 0; e < 8; ++e) ss += x[e] * x[e];
    }
    r = rsqrtf(ss * (1.0f / D) + eps);
  }
  auto scale = [&](int u, float* x) {
    unpack8(raw[u], x);
    if (norm) {
      float wf[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(w) + u), wf);
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] *= r * wf[e];
    }
  };
  if (cosr != nullptr && rope_half) {   // LigerRopeFunction (math.py:27): element i pairs with i + D/2
#pragma unroll
    for (int u = 0; u < U / 2; ++u) {
      float x1[8], x2[8];
      scale(u, x1);
      scale(u + U / 2, x2);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float c = __ldg(cosr + 8 * u + e), sn = __ldg(sinr + 8 * u + e);
        const float a = x1[e], b = x2[e];
        x1[e] = a * c - b * sn;
        x2[e] = b * c + a * sn;
      }
      raw[u] = pack8(x1);
      raw[u + U / 2] = pack8(x2);
    }
  } else if (norm || cosr != nullptr) {
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float x[8];
      scale(u, x);
      if (cosr != nullptr) {   // interleaved pairs (2i, 2i+1) (math.py:60-65)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float c = __ldg(cosr + 4 * u + i), sn = __ldg(sinr + 4 * u + i);
          const float a = x[2 * i], b = x[2 * i + 1];
          x[2 * i] = a * c - b * sn;
          x[2 * i + 1] = b * c + a * sn;
        }
      }
      raw[u] = pack8(x);
    }
  }
}
#endif

}  // namespace osb
