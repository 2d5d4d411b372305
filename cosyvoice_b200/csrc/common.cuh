// Device-side helpers shared by all kernels.
#pragma once
#include "cvk_internal.h"

struct EpiDev {
  const float* bias;
  const float* rowvec;
  int rowvec_ld;
  int act1;
  float act1_param;
  const float* alpha1;
  float scale;
  const float* resid;
  int resid_ld;
  const int* row2seq;
  int accumulate;
  void* out;
  int out_dtype;
  int out_ld;
  int act2;
  float act2_param;
  const float* alpha2;
  void* out2;
  int out2_dtype;
  int out2_ld;
  int ab_f16;        // wgmma GEMM: operands are IEEE half (the .f16 instruction variant) instead of bf16
};

inline EpiDev to_dev(const Epilogue& e) {
  EpiDev d;
  d.bias = e.bias;
  d.rowvec = e.rowvec;
  d.rowvec_ld = e.rowvec_ld;
  d.act1 = e.act1;
  d.act1_param = e.act1_param;
  d.alpha1 = e.alpha1;
  d.scale = e.scale;
  d.resid = e.resid.p ? e.resid.f32() : nullptr;
  d.resid_ld = e.resid.ld;
  d.row2seq = e.row2seq;
  d.accumulate = e.accumulate;
  d.out = e.out.p;
  d.out_dtype = e.out.dtype;
  d.out_ld = e.out.ld;
  d.act2 = e.act2;
  d.act2_param = e.act2_param;
  d.alpha2 = e.alpha2;
  d.out2 = e.out2.p;
  d.out2_dtype = e.out2.dtype;
  d.out2_ld = e.out2.ld;
  d.ab_f16 = 0;
  return d;
}

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f32<bf16>(float v) { return __float2bfloat16_rn(v); }
// saturating: an activation beyond the half range becomes +-65504, not inf (fp32 accumulation downstream stays finite)
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f)); }
// 16-bit storage of either kind as raw bits
__device__ __forceinline__ unsigned short f32_to_16(float v, int dtype) {
  if (dtype == DT_F16) return __half_as_ushort(from_f32<__half>(v));
  return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}
__device__ __forceinline__ float f16bits_to_f32(unsigned short b, int dtype) {
  return dtype == DT_F16 ? __half2float(__ushort_as_half(b)) : __bfloat162float(__ushort_as_bfloat16(b));
}

__device__ __forceinline__ float ld_any(const void* p, int dtype, size_t i) {
  return dtype == DT_F32 ? ((const float*)p)[i] : f16bits_to_f32(((const unsigned short*)p)[i], dtype);
}
__device__ __forceinline__ void st_any(void* p, int dtype, size_t i, float v) {
  if (dtype == DT_F32) ((float*)p)[i] = v;
  else ((unsigned short*)p)[i] = f32_to_16(v, dtype);
}

// torch semantics: F.gelu(approximate='none'), F.silu, F.mish (softplus threshold 20), F.elu(alpha=1),
// F.leaky_relu(slope), Snake (transformer/activation.py:73-84), tanh
__device__ __forceinline__ float apply_act(int act, float x, float param, float alpha) {
  switch (act) {
    case ACT_GELU: return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f));
    case ACT_SILU: return x / (1.f + expf(-x));
    case ACT_MISH: {
      float sp = x > 20.f ? x : log1pf(expf(x));
      return x * tanhf(sp);
    }
    case ACT_ELU: return x > 0.f ? x : expm1f(x);
    case ACT_LRELU: return x > 0.f ? x : x * param;
    case ACT_SNAKE: {
      float s = sinf(x * alpha);
      return x + (1.0f / (alpha + 1e-9f)) * (s * s);
    }
    case ACT_TANH: return tanhf(x);
    case ACT_ABS: return fabsf(x);
    case ACT_GELU_TANH: return 0.5f * x * (1.f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
    default: return x;
  }
}

// bf16-mode variants: hardware approximations (ex2.approx / tanh.approx / sin.approx, fast division).  Their error
// (<= ~1e-6 absolute on O(1) values) is two orders below the bf16 rounding of the stored result.
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_exp(float x) { return fast_ex2(x * 1.4426950408889634f); }
__device__ __forceinline__ float fast_tanh(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float apply_act_fast(int act, float x, float param, float alpha) {
  switch (act) {
    case ACT_GELU: {
      // 0.5 x (1 + erf(x/sqrt2)) with erf(z) = tanh(1.1283792 z + 0.1009114 z^3 + ...) folded into the classic
      // x -> 0.5 x (1 + tanh(0.7978846 (x + 0.044715 x^3))) form on the hardware tanh: max |deviation| from the exact-erf GELU
      // 5e-4, an eighth of a bf16 ulp at |x| ~ 1 (the result is stored as bf16); 6 instructions instead of ~25.
      const float u = x * fmaf(x * x, 0.0356774081f, 0.7978845608f);
      return 0.5f * x * (1.f + fast_tanh(u));
    }
    case ACT_SILU: return __fdividef(x, 1.f + fast_exp(-x));
    case ACT_MISH: {
      // x * tanh(log(1 + e^x)) = x * e(e+2) / (e(e+2) + 2)
      float e = fast_exp(fminf(x, 20.f));
      float n = e * (e + 2.f);
      return x > 20.f ? x : x * __fdividef(n, n + 2.f);
    }
    case ACT_ELU: return x > 0.f ? x : fast_exp(x) - 1.f;
    case ACT_LRELU: return x > 0.f ? x : x * param;
    case ACT_SNAKE: {
      float s = __sinf(x * alpha);
      return fmaf(__fdividef(1.f, alpha + 1e-9f), s * s, x);
    }
    case ACT_TANH: return fast_tanh(x);
    case ACT_ABS: return fabsf(x);
    case ACT_GELU_TANH: {
      const float u = x * fmaf(x * x, 0.0356774081f, 0.7978845608f);
      return 0.5f * x * (1.f + fast_tanh(u));
    }
    default: return x;
  }
}
// 16 values at once: the dispatch on the (run-time) activation kind happens ONCE, outside the element loop.  With the switch
// inside an unrolled loop every element would pay the whole dispatch.
// tanh-form GELU of 16 values with the tanh of TWO arguments per MUFU instruction (tanh.approx.f16x2): the GELU epilogue of
// ff.net.0 is MUFU-bound (one tanh per output element, 16 per clock per SM).  The
// half-precision tanh is off by <= 5e-4 absolute, i.e. <= 2.5e-4 |x| in the GELU - below the bf16 rounding of the stored result
// (3.9e-3 |x|); only the bf16-mode epilogues come here.
__device__ __forceinline__ void gelu16_packed(float* v) {
#pragma unroll
  for (int i = 0; i < 16; i += 2) {
    const float x0 = v[i], x1 = v[i + 1];
    const float u0 = fminf(fmaxf(x0 * fmaf(x0 * x0, 0.0356774081f, 0.7978845608f), -10.f), 10.f);
    const float u1 = fminf(fmaxf(x1 * fmaf(x1 * x1, 0.0356774081f, 0.7978845608f), -10.f), 10.f);
    const __half2 h = __floats2half2_rn(u0, u1);
    uint32_t t;
    asm("tanh.approx.f16x2 %0, %1;" : "=r"(t) : "r"(*reinterpret_cast<const uint32_t*>(&h)));
    const float2 tf = __half22float2(*reinterpret_cast<const __half2*>(&t));
    v[i] = 0.5f * x0 * (1.f + tf.x);
    v[i + 1] = 0.5f * x1 * (1.f + tf.y);
  }
}
__device__ __forceinline__ void act16_fast(int act, float* v, float param, const float* __restrict__ alpha /*per column or null*/) {
  switch (act) {
    case ACT_NONE: break;
    case ACT_GELU:
      gelu16_packed(v);
      break;
    case ACT_SILU:
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = apply_act_fast(ACT_SILU, v[i], 0.f, 1.f);
      break;
    case ACT_MISH:
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = apply_act_fast(ACT_MISH, v[i], 0.f, 1.f);
      break;
    case ACT_ELU:
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = apply_act_fast(ACT_ELU, v[i], 0.f, 1.f);
      break;
    case ACT_LRELU:
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = v[i] > 0.f ? v[i] : v[i] * param;
      break;
    case ACT_SNAKE:
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = apply_act_fast(ACT_SNAKE, v[i], 0.f, alpha ? alpha[i] : 1.f);
      break;
    case ACT_TANH:
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = fast_tanh(v[i]);
      break;
    case ACT_ABS:
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = fabsf(v[i]);
      break;
    case ACT_GELU_TANH:
      gelu16_packed(v);
      break;
    default: break;
  }
}

template <bool FAST>
__device__ __forceinline__ float act_sel(int act, float x, float param, float alpha) {
  return FAST ? apply_act_fast(act, x, param, alpha) : apply_act(act, x, param, alpha);
}

// One output element through the fused epilogue (see struct Epilogue in cvk_internal.h).
template <bool FAST = false>
__device__ __forceinline__ void epi_store(const EpiDev& e, int r, int n, float acc) {
  int seq = 0;
  bool valid = true;
  if (e.row2seq) {
    seq = e.row2seq[r];
    valid = seq >= 0;
  }
  float v = acc;
  if (e.bias) v += e.bias[n];
  if (e.rowvec && valid) v += e.rowvec[(size_t)seq * e.rowvec_ld + n];
  v = act_sel<FAST>(e.act1, v, e.act1_param, e.alpha1 ? e.alpha1[n] : 1.f) * e.scale;
  if (e.resid) v += e.resid[(size_t)r * e.resid_ld + n];
  if (!valid) v = 0.f;
  size_t o = (size_t)r * e.out_ld + n;
  if (e.accumulate) v += ld_any(e.out, e.out_dtype, o);
  st_any(e.out, e.out_dtype, o, v);
  if (e.out2) {
    float w = valid ? act_sel<FAST>(e.act2, v, e.act2_param, e.alpha2 ? e.alpha2[n] : 1.f) : 0.f;
    st_any(e.out2, e.out2_dtype, (size_t)r * e.out2_ld + n, w);
  }
}

// Programmatic dependent launch (PDL): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start
// while its predecessor in the stream is still running.  pdl_trigger() lets the NEXT kernel start launching; pdl_wait() blocks
// until the PREVIOUS kernel has completed and its writes are visible.  Everything before pdl_wait() may only touch data no
// kernel of the chain writes (weights, constants) and may not write global memory.  Both are no-ops in a normal launch.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// chain timeline (debug option chain_timeline): per launch, tl[0] = entry of CTA 0, tl[1] = CTA 0 past pdl_wait, tl[2] = last CTA end
__device__ __forceinline__ void tl_stamp(long long* tl, int which) {
  if (tl == nullptr || threadIdx.x != 0) return;
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  if (which == 2) atomicMax((unsigned long long*)&tl[2], (unsigned long long)t);
  else if (blockIdx.x == 0 && blockIdx.y == 0) tl[which] = t;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// LayerNorm core of a 256-wide row held by one warp, lane l holding columns 4l..4l+3 (v[0..3]) and 128+4l..128+4l+3 (v[4..7]):
// mean, biased variance, eps inside the sqrt, then the optional affine.  Every kernel that normalises the flow estimator's rows
// goes through here, so their results agree bit for bit.
__device__ __forceinline__ void ln256_warp(float* v, const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int c0, int c1) {
  const float mean = warp_sum(((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]))) * (1.f / 256.f);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i] -= mean;
    q = fmaf(v[i], v[i], q);
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.f / 256.f) + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] *= rstd;
  if (gamma) {
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c0), gb = *reinterpret_cast<const float4*>(gamma + c1);
    v[0] *= ga.x; v[1] *= ga.y; v[2] *= ga.z; v[3] *= ga.w; v[4] *= gb.x; v[5] *= gb.y; v[6] *= gb.z; v[7] *= gb.w;
    if (beta) {
      const float4 ba = *reinterpret_cast<const float4*>(beta + c0), bb = *reinterpret_cast<const float4*>(beta + c1);
      v[0] += ba.x; v[1] += ba.y; v[2] += ba.z; v[3] += ba.w; v[4] += bb.x; v[5] += bb.y; v[6] += bb.z; v[7] += bb.w;
    }
  }
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
