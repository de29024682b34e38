// Per-pixel output stage shared by the VarDCT filter store (kernels.cu) and the thumbnail store (modular_kernels.cu):
// XYB -> linear RGB with the re-targeted opsin matrix (render/stages/xyb.rs), the output transfer function
// (render/stages/from_linear.rs) and the sample conversions (render/stages/convert.rs). `Cfg` is any parameter block with
// the FrameDev colour fields: opsin, bias_cbrt, scaled_bias, intensity_scale, output_tf, output_format, tf_gamma,
// tf_lum, tf_hlg_exp and tf_pq_mul.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../../include/jxg.h"

namespace jxgpu {

// convert.rs:574-598: the 32x32 blue-noise dither of u8 outputs. One copy per translation unit.
static __constant__ float c_dither[1024] = {
#include "dither_table.inc"
};

// color/tf.rs:13-44
__device__ __forceinline__ float linear_to_srgb(float v) {
  const float P[5] = {-5.135152395e-4f, 5.287254571e-3f, 3.903842876e-1f, 1.474205315f, 7.352629620e-1f};
  const float Q[5] = {1.004519624e-2f, 3.036675394e-1f, 1.340816930f, 9.258482155e-1f, 2.424867759e-2f};
  float a = fabsf(v), r;
  if (a < 0.0031308f) {
    r = a * 12.92f;
  } else {
    float s = sqrtf(a);
    float yp = P[4], yq = Q[4];
#pragma unroll
    for (int i = 3; i >= 0; i--) {
      yp = fmaf(yp, s, P[i]);
      yq = fmaf(yq, s, Q[i]);
    }
    r = yp / yq;
  }
  return copysignf(r, v);
}

// render/stages/from_linear.rs:56-112: the output transfer function on display-referred linear RGB. The sRGB curve is
// handled by the callers (their hot path); this is the rare-encoding switch, written from color/tf.rs with the device's
// exp2f / log2f where the reference uses its own rational fast_powf (max relative error 3e-5 there).
template <class Cfg>
__device__ __noinline__ void from_linear_other(const Cfg& F, float (&v)[3]) {
  auto rat5 = [](float x, const float* p, const float* q) {
    float yp = p[4], yq = q[4];
#pragma unroll
    for (int i = 3; i >= 0; i--) {
      yp = fmaf(yp, x, p[i]);
      yq = fmaf(yq, x, q[i]);
    }
    return yp / yq;
  };
  switch (F.output_tf) {
    case JXG_TF_GAMMA:
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float a = fabsf(v[c]);
        v[c] = copysignf(a > 0.0f ? exp2f(F.tf_gamma * log2f(a)) : 0.0f, v[c]);
      }
      break;
    case JXG_TF_BT709: {  // tf.rs:114-150
      const float P[5] = {-9.625309705734253e-2f, -2.2635456919670105e-1f, 1.935774803161621e1f, 5.897886276245117e1f, 2.3947298049926758e1f};
      const float Q[5] = {1.0f, 1.877663230895996e1f, 5.5292449951171875e1f, 2.6565317153930664e1f, 3.269049823284149e-1f};
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float a = fabsf(v[c]);
        v[c] = copysignf(a < 0.018f ? a * 4.5f : rat5(sqrtf(a), P, Q), v[c]);
      }
      break;
    }
    case JXG_TF_PQ: {  // tf.rs:236-283
      const float P[5] = {1.351392e-2f, -1.095778f, 5.522776e1f, 1.492516e2f, 4.838434e1f};
      const float Q[5] = {1.012416f, 2.016708e1f, 9.26371e1f, 1.120607e2f, 2.590418e1f};
      const float PS[5] = {9.863406e-6f, 3.881234e-1f, 1.352821e2f, 6.889862e4f, -2.864824e5f};
      const float QS[5] = {3.371868e1f, 1.477719e3f, 1.608477e4f, -4.389884e4f, -2.072546e5f};
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float a = fabsf(v[c]);
        const float a14 = sqrtf(sqrtf(a * F.tf_pq_mul));
        v[c] = copysignf(a < 1e-4f ? rat5(a14, PS, QS) : rat5(a14, P, Q), v[c]);
      }
      break;
    }
    case JXG_TF_HLG: {  // tf.rs:381-395 (inverse OOTF), 481-497 (OETF)
      if (F.tf_hlg_exp != 0.0f) {
        const float mixed = fmaf(v[0], F.tf_lum[0], fmaf(v[1], F.tf_lum[1], v[2] * F.tf_lum[2]));
        float lg;
        if (mixed > 0.0f) {
          lg = log2f(mixed);
        } else {
          // Dark or out-of-gamut pixels. log2f gives NaN here; the reference's fast_log2f (util/fast_math.rs:128-137)
          // splits the bits with wrapping integer arithmetic instead: the exponent of a negative value comes out 256
          // higher (256 lower from |mixed| >= 2/3), the mantissa is that of |mixed|, and +0 comes out as -127.
          const uint32_t bits = __float_as_uint(mixed);
          const int32_t ex = int32_t(bits - 0x3f2aaaabu) >> 23;
          lg = log2f(__uint_as_float(bits - (uint32_t(ex) << 23))) + float(ex);
        }
        const float mult = exp2f(F.tf_hlg_exp * lg);
#pragma unroll
        for (int c = 0; c < 3; c++) v[c] *= mult;
      }
      const float kA = 0.17883277f, kB = 1.0f - 4.0f * 0.17883277f, kC = 0.5599107295f;
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float a = fabsf(v[c]);
        v[c] = copysignf(a <= 1.0f / 12.0f ? sqrtf(3.0f * a) : kA * 0.69314718056f * log2f(12.0f * a - kB) + kC, v[c]);
      }
      break;
    }
    default: break;  // JXG_TF_LINEAR
  }
}

// One XYB sample -> the output encoding's RGB before the sample conversion: opsin inverse (xyb.rs:145-241) and the
// transfer function.
template <class Cfg>
__device__ __forceinline__ void xyb_to_output(const Cfg& F, float vx, float vy, float vb, float (&v)[3]) {
  float l = vy + vx - F.bias_cbrt[0], mm = vy - vx - F.bias_cbrt[1], s = vb - F.bias_cbrt[2];
  float l2 = l * l, m2 = mm * mm, s2 = s * s;
  float sl = l * F.intensity_scale, sm = mm * F.intensity_scale, ss = s * F.intensity_scale;
  l = fmaf(l2, sl, F.scaled_bias[0]);
  mm = fmaf(m2, sm, F.scaled_bias[1]);
  s = fmaf(s2, ss, F.scaled_bias[2]);
  v[0] = fmaf(F.opsin[0], l, fmaf(F.opsin[1], mm, F.opsin[2] * s));
  v[1] = fmaf(F.opsin[3], l, fmaf(F.opsin[4], mm, F.opsin[5] * s));
  v[2] = fmaf(F.opsin[6], l, fmaf(F.opsin[7], mm, F.opsin[8] * s));
  if (F.output_tf == JXG_TF_SRGB) {
#pragma unroll
    for (int c = 0; c < 3; c++) v[c] = linear_to_srgb(v[c]);
  } else if (F.output_tf != JXG_TF_LINEAR) {
    from_linear_other(F, v);
  }
}

// 16-bit stores of one colour sample. U16: ConvertF32ToU16Stage (convert.rs:739-762: clamp to [0, 1], scale by
// 2^16 - 1, round to nearest, ties to even like the AVX2 store). F16: ConvertF32ToF16Stage (convert.rs:831-857) with the
// clamp range frame/render.rs:746-750 gives PQ and HLG outputs.
template <class Cfg>
__device__ __forceinline__ uint16_t sample16(const Cfg& F, float v) {
  if (F.output_format == JXG_FORMAT_RGB_U16) return uint16_t(__float2int_rn(fminf(fmaxf(v, 0.0f), 1.0f) * 65535.0f));
  if (F.output_tf == JXG_TF_PQ) v = fminf(fmaxf(v, 0.0f), 1.0f);
  else if (F.output_tf == JXG_TF_HLG) v = fminf(fmaxf(v, -0.074f), 1.1f);
  // util/float16.rs:82-141: round to nearest even for normal halves, but the reference TRUNCATES into the subnormal range
  // (and shifts one bit too far: 2^-15 becomes 2^-16 - reproduced, identical output is the contract)
  const uint32_t bits = __float_as_uint(v), mag = bits & 0x7fffffffu;
  if (mag < 0x38800000u) {  // |v| < 2^-14
    const uint32_t sign = (bits >> 16) & 0x8000u;
    const int unbiased = int(mag >> 23) - 127;
    if ((mag >> 23) == 0 || unbiased < -24) return uint16_t(sign);
    return uint16_t(sign | (((mag & 0x007fffffu) | 0x00800000u) >> (uint32_t(-14 - unbiased) + 14)));
  }
  return __half_as_ushort(__float2half_rn(v));
}

// u8 store of colour sample c at coded pixel (x, y): the blue-noise dither, clamp and round (convert.rs:574-598).
__device__ __forceinline__ uint8_t sample8(float v, int x, int y, int c) {
  const float dth = c_dither[((y + 13 * c) & 31) * 32 + ((x + 23 * c) & 31)];
  const float sc = fminf(fmaxf(v * 255.0f + dth, 0.0f), 255.0f);
  return uint8_t(__float2int_rn(sc));
}

}  // namespace jxgpu
