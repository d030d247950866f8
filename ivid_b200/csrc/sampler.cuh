// Fused denoising-step kernels: classifier-free-guidance mix + DDPM / DDIM / DPM-Solver++(2M) / UniPC update (+ multiview
// replace/constrain guidance) in ONE HBM pass over [N,4,H,W], coefficients read from a device-resident table and step
// state (no per-step H2D).
//   reference: ClassifierFreeGuidance.model_inference classifier_free_guidance.py:39-42
//              DdpmSampler.p_mean_variance / sample_once   samplers/ddpm.py:85-100,127-131
//              DdimSampler.sample_once                      samplers/ddim.py:81-103
//              DPM-Solver++(2M), data-prediction multistep  Lu et al. 2022, arXiv:2211.01095 (no reference counterpart)
//              UniPC, bh2 predictor-corrector               Zhao et al. 2023, arXiv:2302.04867 (no reference counterpart)
//              adaptive projected guidance                  Sadat et al. 2025, arXiv:2410.02416 (no reference counterpart)
//              InpaintCFG.make_cond_inputs                  frameworks/inpaint_cfg.py:33-49
//              SuperResCFG.make_cond_inputs                 frameworks/sr_cfg.py:31-36
#pragma once
#include <type_traits>

#include "common.cuh"

namespace ivid {

// ----------------------------------------------------------------------------------------------
// Philox4x32-10 counter RNG + Box-Muller (in-kernel N(0,1) for the production path; parity tests inject noise).
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}
__device__ __forceinline__ float u01(uint32_t x) { return (static_cast<float>(x) + 0.5f) * 2.3283064365386963e-10f; }
// four N(0,1) draws for (seed, stream, idx)
__device__ __forceinline__ float4 philox_normal4(uint64_t seed, uint32_t stream, uint32_t idx) {
  const uint4 r = philox4x32_10(make_uint4(idx, stream, 0u, 0u),
                                make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)));
  const float r0 = sqrtf(-2.0f * logf(u01(r.x))), a0 = 6.283185307179586f * u01(r.y);
  const float r1 = sqrtf(-2.0f * logf(u01(r.z))), a1 = 6.283185307179586f * u01(r.w);
  float s0, c0, s1, c1;
  sincosf(a0, &s0, &c0);
  sincosf(a1, &s1, &c1);
  return make_float4(r0 * c0, r0 * s0, r1 * c1, r1 * s1);
}

// Per-timestep coefficient row (fp32 casts of the reference's float64 numpy tables).
struct StepCoef {
  float sqrt_recip_acp;      // sqrt(1/acp[t])
  float sqrt_recipm1_acp;    // sqrt(1/acp[t] - 1)
  float post_mean_coef1;     // DDPM
  float post_mean_coef2;     // DDPM
  float post_logvar;         // DDPM posterior_log_variance_clipped[t]
  float acp;                 // alphas_cumprod[t]
  float acp_prev;            // alphas_cumprod_prev[t]  (acp_prev[0] = 1)
  float pad;
};

struct GuideParams {           // DDIM multiview guidance (all maps fp32 NCHW, nullptr = disabled)
  const float* rgb;            // [N,3,H,W]
  const float* rgb_mask;       // [N,1,H,W]
  const float* depth;          // [N,1,H,W]
  const float* depth_mask;     // [N,1,H,W]
  const float* convex;         // [N,1,H,W]
  float w_rgb, w_rgb_c;        // w and (1-w) as the reference's python floats cast to fp32
  float w_depth, w_depth_c;
  float w_convex, w_convex_c;
};

// Step kinds (template argument of the step kernels; ivid_step_args_t.kind)
constexpr int kStepDdpm = 0, kStepDdim = 1, kStepDpm = 2;

// DPM-Solver++ per-step scalars, computed in double by the step-state kernel and rounded to fp32 (sampler.cu):
//   x_p = c_xt * x_t - c_d * D (+ c_z * z),  D = D0 (order 1) or w0 * D0 + w1 * D_{-1} (order 2)
struct DpmStep {
  float c_xt;                  // ODE: sigma_p / sigma_s;             SDE: sigma_p / sigma_s * exp(-h)
  float c_d;                   // ODE: alpha_p * (exp(-h) - 1);       SDE: alpha_p * (exp(-2h) - 1)
  float w0, w1;                // 1 + 1/(2r), -1/(2r)
  int order;                   // 1 or 2
  float c_z;                   // ODE: 0;                             SDE: sigma_p * sqrt(1 - exp(-2h)), 0 on the final step
};

// UniPC per-step coefficients (include/ivid_b200.h), computed in double by the step-state kernel and rounded to fp32 once
// (sampler.cu: unipc_step_state), folded into two linear combinations over the step's planes, D0 = D_i and the history
// H_j = D_{i-j}:
//   corrector (corr_order >= 1):  x^c = a * base + v[0] * D0 + v[1] * H_1 + ... + v[corr_order] * H_corr_order
//                 (corr_order 0):  x^c = x_t
//   predictor:                    x_p = c * x^c + w[0] * D0 + w[1] * H_1 + ... + w[order - 1] * H_{order-1}
// Only the terms of the two orders are evaluated: the history beyond them may hold anything.
struct UniPcStep {
  float a, v[4];
  float c, w[3];
  int corr_order;              // 0 (first step: no corrector) .. 3
  int order;                   // predictor order 1..3 (1 on the final step, where c = 0, w[0] = 1: x_p = D0)
};

struct StepParams {
  const float* x_t;            // [N,C,H,W]
  const float* noise;          // [N,C,H,W] injected N(0,1) or nullptr -> Philox
  float* x_prev;               // [N,C,H,W]
  float* pred_x0;              // optional
  const StepCoef* table;       // [T]
  const int* t_index;          // device scalar: table row for the model timestep (t for DDPM, t-1 for DDIM)
  const int* t_prev;           // DDIM: device scalar t_prev (acp_prev row); DDPM: unused
  int N, C, HW;
  int cfg;                     // 1: eps = (1+s)*eps_c - s*eps_u;  2: eps = (1+s)*eps_c (strength <= 0: no null-class forward)
  float strength;
  int clip;
  float eta;
  uint64_t seed;
  uint32_t stream;             // Philox stream id (step counter supplied by caller) when noise == nullptr
  const int* stream_dev;       // optional device step counter added to `stream`
  GuideParams g;
  // DPM-Solver++ only (appended, so the DDPM / DDIM layout is unchanged)
  const DpmStep* dpm;          // device step state
  float* hist;                 // [N,C,H,W] D_{-1} on entry (order 2), overwritten in place with this step's D0
  // guidance interval on the device-timestep route (appended): device flag, 0 = this step is unguided, so eps = eps_c
  // whatever cfg says (the null-class rows are ignored); nullptr = always guided
  const int* guided;
  // perturbed-attention guidance (appended): 1 = the eps rows hold a third block, the forward with identity attention maps,
  // after the conditional (and, at cfg 1, the null-class) rows, and eps gains pag_scale * (eps_c - eps_perturbed)
  int pag;
  float pag_scale;
};

// (1 + strength) * eps_c - strength * eps_u (only evaluated with strength > 0).  Every product / sum of the step arithmetic is
// written with explicit round-to-nearest intrinsics (no compiler-chosen FMA contraction), so that the instantiations of
// step_kernel - the same formulas inlined behind different sources of eps - produce identical bits.
__device__ __forceinline__ float cfg_mix(float ec, float eu, float strength) {
  return __fsub_rn(__fmul_rn(__fadd_rn(1.0f, strength), ec), __fmul_rn(strength, eu));
}
// the guidance of this step: p.cfg in bits 0-1 and kPagBit when the perturbed-attention term applies; 0 when the device
// flag says the step lies outside the guidance interval (which gates both guidances)
constexpr int kPagBit = 4;
__device__ __forceinline__ int step_cfg(const StepParams& p) {
  return (p.guided != nullptr && *p.guided == 0) ? 0 : (p.cfg | (p.pag ? kPagBit : 0));
}
// row block of the perturbed eps: after the conditional rows, and after the null-class rows when cfg & 3 == 1
__device__ __forceinline__ int pag_block(int cfg) { return (cfg & 3) == 1 ? 2 : 1; }
// the guidance-mixed eps of four elements, cfg = step_cfg(p): eps(b, e) loads row block b of eps: 0 the conditional rows,
// 1 the null-class rows (called only when cfg & 3 == 1), pag_block(cfg) the perturbed rows (only with kPagBit).  The
// classifier-free part G is formed first, then G + pag_scale * (eps_c - eps_perturbed), each operation rounded on its own.
// eps_c is loaded again for the PAG term rather than kept live across G (the same bits: every source is deterministic).  The
// step kernels take the term as a compile-time switch (step_kernel's kPag): without it cfg & kPagBit is known to be 0, the
// branch is not compiled, and the steps without PAG keep the code they had before it existed.
template <typename Eps>
__device__ __forceinline__ void mix_eps4(const StepParams& p, int cfg, Eps&& eps, float (&e)[4]) {
  eps(0, e);
  if ((cfg & 3) == 1) {
    float eu[4];
    eps(1, eu);
#pragma unroll
    for (int j = 0; j < 4; ++j) e[j] = cfg_mix(e[j], eu[j], p.strength);
  } else if ((cfg & 3) == 2) {
#pragma unroll
    for (int j = 0; j < 4; ++j) e[j] = __fmul_rn(__fadd_rn(1.0f, p.strength), e[j]);
  }
  if (cfg & kPagBit) {
    float ec[4], ep[4];
    eps(0, ec);
    eps(pag_block(cfg), ep);
#pragma unroll
    for (int j = 0; j < 4; ++j) e[j] = __fadd_rn(e[j], __fmul_rn(p.pag_scale, __fsub_rn(ec[j], ep[j])));
  }
}

// the whole guidance mix of the step alone (framework.model_inference with perturbed-attention guidance): out = mix_eps4 over
// the row blocks of eps, n4 quads each; p carries cfg, strength, pag and pag_scale
__global__ void __launch_bounds__(256) guidance_mix_kernel(const float* __restrict__ eps, float* __restrict__ out, size_t n4,
                                                           const StepParams p) {
  const int cfg = step_cfg(p);
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float e[4];
    mix_eps4(p, cfg, [&](int b, float (&v)[4]) {
      const float4 t = ldg_f4(eps + (b * n4 + i) * 4);
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }, e);
    stg_f4(out + 4 * i, make_float4(e[0], e[1], e[2], e[3]));
  }
}

// classifier-free-guidance mix alone (framework.model_inference): out = (1+s)*eps[0:n) - s*eps[n:2n)
__global__ void __launch_bounds__(256) cfg_mix_kernel(const float* __restrict__ eps2, float* __restrict__ out, size_t n4, float strength) {
  const float4* a = reinterpret_cast<const float4*>(eps2);
  const float4* b = a + n4;
  float4* o = reinterpret_cast<float4*>(out);
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 c = __ldg(a + i), u = __ldg(b + i);
    o[i] = make_float4((1.0f + strength) * c.x - strength * u.x, (1.0f + strength) * c.y - strength * u.y,
                       (1.0f + strength) * c.z - strength * u.z, (1.0f + strength) * c.w - strength * u.w);
  }
}

// Philox stream of the forward diffusion's noise: no step uses it (steps use their index, below T)
constexpr uint32_t kDiffuseStream = 0xFFFFFFFFu;

// q(x_t | x_0): out = a * x0 + b * z with a = fp32(sqrt(acp[t])), b = fp32(sqrt(1 - acp[t])), rounded as the reference's two
// fp32 tensor products and their sum (no FMA).  z is the injected noise, or Philox(seed, kDiffuseStream) indexed by quad as
// the step kernels index their noise.
__global__ void __launch_bounds__(256) diffuse_kernel(const float* __restrict__ x0, const float* __restrict__ noise,
                                                      float* __restrict__ out, size_t n4, float a, float b, uint64_t seed) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 z = noise != nullptr ? ldg_f4(noise + 4 * i) : philox_normal4(seed, kDiffuseStream, static_cast<uint32_t>(i));
    const float4 x = ldg_f4(x0 + 4 * i);
    stg_f4(out + 4 * i, make_float4(__fadd_rn(__fmul_rn(a, x.x), __fmul_rn(b, z.x)), __fadd_rn(__fmul_rn(a, x.y), __fmul_rn(b, z.y)),
                                    __fadd_rn(__fmul_rn(a, x.z), __fmul_rn(b, z.z)), __fadd_rn(__fmul_rn(a, x.w), __fmul_rn(b, z.w))));
  }
}

// Per-step scalars derived once per thread from the device-resident step state.
struct StepScalars {
  StepCoef k;
  float nz;          // DDPM: t != 0 ; DDIM / DPM: t_prev != 0
  float sd;          // DDPM: exp(0.5 * posterior_log_variance_clipped)
  float sigma, c_x0, c_eps;    // DDIM
  DpmStep d;                   // DPM-Solver++
  uint32_t stream;
};
// whether the step draws N(0,1) noise (DPM-Solver++: only the SDE variant, and not on its final step)
template <int kKind>
__device__ __forceinline__ bool step_draws_noise(const StepScalars& s) {
  return kKind == kStepDdpm || (kKind == kStepDdim && s.sigma != 0.0f) || (kKind == kStepDpm && s.d.c_z != 0.0f);
}
template <int kKind>
__device__ __forceinline__ StepScalars step_scalars(const StepParams& p) {
  StepScalars s;
  s.k = p.table[*p.t_index];
  s.stream = p.stream + (p.stream_dev ? static_cast<uint32_t>(*p.stream_dev) : 0u);
  if (kKind == kStepDpm) {
    s.nz = (*p.t_prev != 0) ? 1.0f : 0.0f;
    s.d = *p.dpm;
    s.sigma = 0.f; s.c_x0 = 0.f; s.c_eps = 0.f; s.sd = 0.f;
  } else if (kKind == kStepDdpm) {
    s.nz = (*p.t_index != 0) ? 1.0f : 0.0f;
    s.sd = expf(__fmul_rn(0.5f, s.k.post_logvar));
    s.sigma = 0.f; s.c_x0 = 0.f; s.c_eps = 0.f;
  } else {
    const int tprev = *p.t_prev;
    s.nz = (tprev != 0) ? 1.0f : 0.0f;
    const float ab = s.k.acp;
    const float abp = (tprev == 0) ? 1.0f : p.table[tprev - 1].acp;   // alphas_cumprod_prev[t_prev]
    s.sigma = __fmul_rn(__fmul_rn(p.eta, sqrtf(__fdiv_rn(__fsub_rn(1.0f, abp), __fsub_rn(1.0f, ab)))), sqrtf(__fsub_rn(1.0f, __fdiv_rn(ab, abp))));
    s.c_x0 = sqrtf(abp);
    s.c_eps = sqrtf(__fsub_rn(__fsub_rn(1.0f, abp), __fmul_rn(s.sigma, s.sigma)));
    s.sd = 0.f;
  }
  return s;
}
// x_0 = sqrt(1/acp) * x_t - sqrt(1/acp - 1) * eps of one element (before clipping or thresholding)
__device__ __forceinline__ float step_x0(const StepCoef& k, float xt, float e) {
  return __fsub_rn(__fmul_rn(k.sqrt_recip_acp, xt), __fmul_rn(k.sqrt_recipm1_acp, e));
}
// x_0 of one element from x_t and the (already guidance-mixed) eps, clipped to [-1, 1] when p.clip is set
__device__ __forceinline__ float eps_x0(const StepParams& p, const StepCoef& k, float xt, float e) {
  float x0 = step_x0(k, xt, e);
  if (p.clip) x0 = fminf(fmaxf(x0, -1.0f), 1.0f);
  return x0;
}
// dynamic thresholding of one element of x_0 with its sample's s (see threshold_select_kernel)
__device__ __forceinline__ float threshold_x0(float x0, float s) { return __fdiv_rn(fminf(fmaxf(x0, -s), s), s); }
// the replace / constrain guidance of DDIM, DPM-Solver++ and UniPC on x_0 of one element (sample n, channel c, pixel pix);
// nz = (t_prev != 0)
__device__ __forceinline__ float guide_x0(const StepParams& p, float nz, int n, int c, size_t pix, float x0) {
  auto mul = [](float a, float b) { return __fmul_rn(a, b); };
  auto add = [](float a, float b) { return __fadd_rn(a, b); };
  auto sub = [](float a, float b) { return __fsub_rn(a, b); };
  if (c < 3) {
    if (p.g.rgb != nullptr) {
      const float y = p.g.rgb[(static_cast<size_t>(n) * 3 + c) * p.HW + pix];
      const float m = p.g.rgb_mask[static_cast<size_t>(n) * p.HW + pix];
      x0 = add(mul(sub(1.0f, nz), x0), mul(nz, add(mul(add(mul(p.g.w_rgb, y), mul(p.g.w_rgb_c, x0)), m), mul(x0, sub(1.0f, m)))));
    }
  } else if (p.g.depth != nullptr) {
    const float y = p.g.depth[static_cast<size_t>(n) * p.HW + pix];
    const float m = p.g.depth_mask[static_cast<size_t>(n) * p.HW + pix];
    x0 = add(mul(add(mul(p.g.w_depth, y), mul(p.g.w_depth_c, x0)), m), mul(x0, sub(1.0f, m)));
    if (p.g.convex != nullptr) {
      const float cv = p.g.convex[static_cast<size_t>(n) * p.HW + pix];
      x0 = add(mul(x0, m), mul(add(mul(p.g.w_convex, fmaxf(x0, cv)), mul(p.g.w_convex_c, x0)), sub(1.0f, m)));
    }
  }
  return x0;
}
// x_{t-1} and x_0 of one element (sample n, channel c, pixel pix) from x_t, its x_0 after clipping or thresholding and the N(0,1)
// draw z: the replace / constrain guidance, then the DDPM / DDIM / DPM-Solver++ update.  DPM-Solver++: z is read only by the SDE
// variant (c_z != 0), dprev is D_{-1} of the element (read only at order 2) and x0o the guided D0.
template <int kKind>
__device__ __forceinline__ void step_update(const StepParams& p, const StepScalars& s, int n, int c, size_t pix, float xt, float x0,
                                            float z, float dprev, float& xo, float& x0o) {
  const StepCoef& k = s.k;
  auto mul = [](float a, float b) { return __fmul_rn(a, b); };
  auto add = [](float a, float b) { return __fadd_rn(a, b); };
  auto sub = [](float a, float b) { return __fsub_rn(a, b); };
  if (kKind == kStepDdpm) {
    const float mean = add(mul(k.post_mean_coef1, x0), mul(k.post_mean_coef2, xt));
    xo = add(mean, mul(mul(s.nz, s.sd), z));
    x0o = x0;
    return;
  }
  x0 = guide_x0(p, s.nz, n, c, pix, x0);
  if (kKind == kStepDpm) {
    // D_{-1} is not read at order 1: the history may hold anything (first step of a run)
    const float d = s.d.order == 2 ? add(mul(s.d.w0, x0), mul(s.d.w1, dprev)) : x0;
    xo = sub(mul(s.d.c_xt, xt), mul(s.d.c_d, d));
    if (s.d.c_z != 0.0f) xo = add(xo, mul(s.d.c_z, z));    // SDE noise; the ODE expression above keeps its bits
    x0o = x0;
    return;
  }
  const float e2 = __fdiv_rn(sub(mul(k.sqrt_recip_acp, xt), x0), k.sqrt_recipm1_acp);
  const float mean = add(mul(s.c_x0, x0), mul(s.c_eps, e2));
  xo = add(mean, mul(mul(s.nz, s.sigma), z));
  x0o = x0;
}
// the four N(0,1) draws of elements [i, i+4) of the flattened [N,C,H,W] tensor (i % 4 == 0): injected or Philox(seed, stream, i/4)
__device__ __forceinline__ void step_noise4(const StepParams& p, const StepScalars& s, size_t i, bool needed, float (&z)[4]) {
  z[0] = z[1] = z[2] = z[3] = 0.f;
  if (!needed) return;
  const float4 t = p.noise != nullptr ? ldg_f4(p.noise + i) : philox_normal4(p.seed, s.stream, static_cast<uint32_t>(i >> 2));
  z[0] = t.x; z[1] = t.y; z[2] = t.z; z[3] = t.w;
}

// DPM-Solver++ history of elements [i, i+4): D_{-1} before the step (only at order 2; every thread reads and then overwrites
// its own elements, so the buffer is updated in place)
template <int kKind>
__device__ __forceinline__ void hist_load4(const StepParams& p, const StepScalars& s, size_t i, float (&h)[4]) {
  h[0] = h[1] = h[2] = h[3] = 0.f;
  if (kKind != kStepDpm || s.d.order != 2) return;
  const float4 t = *reinterpret_cast<const float4*>(p.hist + i);
  h[0] = t.x; h[1] = t.y; h[2] = t.z; h[3] = t.w;
}
template <int kKind>
__device__ __forceinline__ void hist_store4(const StepParams& p, size_t i, const float (&x0o)[4]) {
  if (kKind == kStepDpm) stg_f4(p.hist + i, make_float4(x0o[0], x0o[1], x0o[2], x0o[3]));
}

// ----------------------------------------------------------------------------------------------
// The step kernel: a source (where x_0 comes from) feeding a sink (what the pass writes).  A source knows its grid-stride work
// unit and, for each quad of the unit (four consecutive pixels of one (n, c) plane), calls f(q, load); load(xt, x0) yields the
// quad's x_t and its guided x_0, clipped or thresholded.  Sinks call load after their loads that do not depend on it (noise,
// history), so the inputs of x_0 do not occupy registers across the Philox draw.  step_kernel<Src, Update<kind>> is a whole
// step; a thresholded step is step_kernel<Src, StoreX0>, threshold_select_kernel, step_kernel<ThresholdedX0, Update<kind>>.
// All share the element arithmetic above, so every route gives the same bits.
// ----------------------------------------------------------------------------------------------
struct Quad {
  size_t i;                    // flat index of the first element in [N,C,H,W] (i % 4 == 0): Philox index i >> 2
  size_t pix;                  // its pixel in the plane
  int n, c;
};
// quad u of the flattened [N,C,H,W] tensor
__device__ __forceinline__ Quad flat_quad(const StepParams& p, size_t u) {
  Quad q;
  q.i = u * 4;
  const int plane = static_cast<int>(q.i / p.HW);      // n*C + c
  q.n = plane / p.C;
  q.c = plane % p.C;
  q.pix = q.i - static_cast<size_t>(plane) * p.HW;
  return q;
}

// What a source makes of the eps row blocks of a quad.  GuidedX0 (every step): the guided, clipped x_0 of each element, from
// mix_eps4.  ApgInputs (the first pass of an APG step, below): the three inputs of adaptive projected guidance.  mix() runs
// before x_t is read, x0() per element after.
struct GuidedX0 {
  using Eps = float[1][4];
  using Out = float[4];
  template <typename Ld>
  __device__ __forceinline__ static void mix(const StepParams& p, int cfg, Ld&& eps, Eps& e) { mix_eps4(p, cfg, eps, e[0]); }
  __device__ __forceinline__ static void x0(const StepParams& p, const StepCoef& k, int j, float xt, const Eps& e, Out& o) {
    o[j] = eps_x0(p, k, xt, e[0][j]);
  }
};

// ----------------------------------------------------------------------------------------------
// Adaptive projected guidance (APG; Sadat, Hilliges, Weber, ICLR 2025, arXiv:2410.02416), per sample n over its M = C*H*W
// elements, on a step with the classifier-free mix (include/ivid_b200.h):
//   D_c = x_0 of eps_c, D_u = x_0 of eps_u, m = (D_c - D_u) + beta * m_prev, c = min(1, r / |m|),
//   k = (1 - eta) <m, D_c> / max(|D_c|^2, tiny), D = D_c + s c (m - k D_c) (+ the PAG term w (D_c - D_p)).
// A step in this mode runs step_kernel<Src, ApgStore> (D_c, m and the PAG term into sampler-owned planes, from HeadTaps on
// the fused route and EpsRows on the separate one), apg_reduce_kernel (the two scalars of every sample) and
// step_kernel<ApgX0, sink> (D, then the update, or StoreX0 and the dynamic threshold).  Both routes share the last two.
// ----------------------------------------------------------------------------------------------
struct ApgParams {
  float* dc;                   // [N,C,H,W] D_c
  float* m;                    // [N,C,H,W] m_prev on entry, m after the first pass (in place)
  float* pag;                  // [N,C,H,W] the PAG term w (D_c - D_p) (steps with PAG only)
  float* scal;                 // [N][2]: fp32(s * c) and fp32(s * c * k)
  float beta;                  // momentum, rounded to fp32 once
  double eta, norm;            // parallel weight and norm bound r (0: no bound), used in double
};
// the momentum update of one element: m = delta + beta * m_prev (beta = 0: m = delta, m_prev is not read)
__device__ __forceinline__ float apg_momentum(float delta, float beta, float m_prev) {
  return beta != 0.0f ? __fadd_rn(delta, __fmul_rn(beta, m_prev)) : delta;
}
// the guided x_0 of one element: D_c + (s c * m - s c k * D_c)
__device__ __forceinline__ float apg_guide(float dc, float m, float sc, float sck) {
  return __fadd_rn(dc, __fsub_rn(__fmul_rn(sc, m), __fmul_rn(sck, dc)));
}
// The first pass's inputs of an element: o[0] = D_c = x_0 of eps_c (never clipped), o[1] = D_c - D_u, o[2] = the PAG term
// w (D_c - D_p).  The differences are taken in eps, where the x_t terms cancel: D_c - D_u = sqrt(1/acp - 1) (eps_u - eps_c)
// and D_c - D_p = sqrt(1/acp - 1) (eps_p - eps_c).  On a step the device flag leaves unguided (cfg 0) only o[0] is formed.
struct ApgInputs {
  using Eps = float[3][4];     // eps_c, eps_u - eps_c, w (eps_p - eps_c)
  using Out = float[3][4];
  template <typename Ld>
  __device__ __forceinline__ static void mix(const StepParams& p, int cfg, Ld&& eps, Eps& e) {
    eps(0, e[0]);
#pragma unroll
    for (int j = 0; j < 4; ++j) e[1][j] = e[2][j] = 0.f;
    if ((cfg & 3) == 1) {
      eps(1, e[1]);
#pragma unroll
      for (int j = 0; j < 4; ++j) e[1][j] = __fsub_rn(e[1][j], e[0][j]);
    }
    if (cfg & kPagBit) {
      eps(pag_block(cfg), e[2]);
#pragma unroll
      for (int j = 0; j < 4; ++j) e[2][j] = __fmul_rn(p.pag_scale, __fsub_rn(e[2][j], e[0][j]));
    }
  }
  __device__ __forceinline__ static void x0(const StepParams&, const StepCoef& k, int j, float xt, const Eps& e, Out& o) {
    o[0][j] = step_x0(k, xt, e[0][j]);
    o[1][j] = __fmul_rn(k.sqrt_recipm1_acp, e[1][j]);
    o[2][j] = __fmul_rn(k.sqrt_recipm1_acp, e[2][j]);
  }
};

// x_0 from the eps buffer [N, 2N or 3N][C,H,W]: rows [0,N) conditional, then [N,2N) unconditional when cfg & 3 == 1, then the
// perturbed rows with kPagBit.  One quad per unit.
struct EpsRows {
  const float* eps;
  __host__ __device__ size_t units(const StepParams& p) const { return static_cast<size_t>(p.N) * p.C * p.HW / 4; }
  template <typename R = GuidedX0, typename F>
  __device__ __forceinline__ void quads(const StepParams& p, const StepCoef& k, int cfg, size_t u, F&& f) const {
    const size_t total = static_cast<size_t>(p.N) * p.C * p.HW;
    const Quad q = flat_quad(p, u);
    f(q, [&](float (&xt)[4], typename R::Out& x0) {
      typename R::Eps e;
      R::mix(p, cfg, [&](int b, float (&v)[4]) {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = eps[b * total + q.i + j];
      }, e);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        xt[j] = p.x_t[q.i + j];
        R::x0(p, k, j, xt[j], e, x0);
      }
    });
  }
};

// x_0 from the tap columns Y of the output head's 1x1 GEMM: eps is the shift-and-add of eps_gather_kernel (same summation
// order), never written to HBM.  One unit = 4 consecutive pixels (one row segment) of one sample, all Co = 4 channels: 4 quads.
struct HeadTaps {
  const float* Y;              // [N, 2N or 3N][H][W][ldy] tap columns (tap*Co + c), row blocks as EpsRows
  const float* bias;           // [Co]
  int H, W, ldy;
  __host__ __device__ size_t units(const StepParams& p) const { return static_cast<size_t>(p.N) * H * (W / 4); }
  // eps of pixel (x, y) of row n (row block n / N, as EpsRows), all 4 channels
  __device__ __forceinline__ void eps4(int n, int y, int x, float (&e)[4]) const {
    e[0] = e[1] = e[2] = e[3] = 0.f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int hh = y + tap / 3 - 1, ww = x + tap % 3 - 1;
      if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
      const float4 v = ldg_f4(Y + ((static_cast<size_t>(n) * H + hh) * W + ww) * ldy + tap * 4);
      e[0] += v.x; e[1] += v.y; e[2] += v.z; e[3] += v.w;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) e[c] += __ldg(bias + c);
  }
  template <typename R = GuidedX0, typename F>
  __device__ __forceinline__ void quads(const StepParams& p, const StepCoef& k, int cfg, size_t g, F&& f) const {
    const int w4 = W / 4;
    const int xg = static_cast<int>(g % w4);
    const int y = static_cast<int>((g / w4) % H);
    const int n = static_cast<int>(g / (static_cast<size_t>(w4) * H));
    typename R::Eps e[4];           // [pixel][block][channel]
#pragma unroll
    for (int j = 0; j < 4; ++j)
      R::mix(p, cfg, [&](int b, float (&v)[4]) { eps4(n + b * p.N, y, xg * 4 + j, v); }, e[j]);
    const size_t pix = static_cast<size_t>(y) * W + xg * 4;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      Quad q;
      q.i = (static_cast<size_t>(n) * 4 + c) * p.HW + pix;
      q.pix = pix;
      q.n = n;
      q.c = c;
      f(q, [&](float (&xt)[4], typename R::Out& x0) {
        const float4 v = ldg_f4(p.x_t + q.i);
        xt[0] = v.x; xt[1] = v.y; xt[2] = v.z; xt[3] = v.w;
        typename R::Eps ec;          // channel c of the four pixels
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int b = 0; b < static_cast<int>(sizeof(ec) / sizeof(ec[0])); ++b) ec[b][j] = e[j][b][c];
#pragma unroll
        for (int j = 0; j < 4; ++j) R::x0(p, k, j, xt[j], ec, x0);
      });
    }
  }
};

// x_0 from a [N,C,H,W] buffer of x_0 before thresholding and s [N] from threshold_select_kernel.  One quad per unit.
struct ThresholdedX0 {
  const float* x0;
  const float* s;
  __host__ __device__ size_t units(const StepParams& p) const { return static_cast<size_t>(p.N) * p.C * p.HW / 4; }
  template <typename F>
  __device__ __forceinline__ void quads(const StepParams& p, const StepCoef&, int, size_t u, F&& f) const {
    const Quad q = flat_quad(p, u);
    const float sn = s[q.n];
    f(q, [&](float (&xt)[4], float (&th)[4]) {
      const float4 v = ldg_f4(x0 + q.i);
      const float x0v[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        xt[j] = p.x_t[q.i + j];
        th[j] = threshold_x0(x0v[j], sn);
      }
    });
  }
};

// x_{t-1}, pred_x0 and the DPM-Solver++ history of a quad: the noise, the history read before it is overwritten (same thread)
// and the replace / constrain guidance + update of step kind kKind
template <int kKind>
struct Update {
  using Scalars = StepScalars;
  __device__ __forceinline__ static StepScalars scalars(const StepParams& p) { return step_scalars<kKind>(p); }
  template <typename Load>
  __device__ __forceinline__ void operator()(const StepParams& p, const StepScalars& s, const Quad& q, Load&& load) const {
    float z[4], hp[4];
    step_noise4(p, s, q.i, step_draws_noise<kKind>(s), z);
    hist_load4<kKind>(p, s, q.i, hp);
    float xt[4], x0[4], xo[4], x0o[4];
    load(xt, x0);
#pragma unroll
    for (int j = 0; j < 4; ++j) step_update<kKind>(p, s, q.n, q.c, q.pix + j, xt[j], x0[j], z[j], hp[j], xo[j], x0o[j]);
    stg_f4(p.x_prev + q.i, make_float4(xo[0], xo[1], xo[2], xo[3]));
    if (p.pred_x0) stg_f4(p.pred_x0 + q.i, make_float4(x0o[0], x0o[1], x0o[2], x0o[3]));
    hist_store4<kKind>(p, q.i, x0o);
  }
};

// The UniPC update of a quad (kind 2 with unipc = 1): corrector, predictor and the shift of the history, in place.  The
// arena holds kUniPcPlanes planes of [N,C,H,W]: the history H_1 .. H_3 (D_{i-1} .. D_{i-3}) and the corrector's base.  Each
// thread reads every plane of its elements before it writes them, so no other thread sees a plane half shifted.  depth =
// the history planes a run keeps (its order); the pointers stay fixed across a run, so consecutive steps replay one graph.
constexpr int kUniPcPlanes = 4;
struct UniPcUpdate {
  float* arena;                // planes 0..2: H_1..H_3, plane 3: base
  size_t plane;                // elements per plane (N*C*H*W)
  float* corrected;            // optional: x^c
  const UniPcStep* u;          // device step state
  int depth;                   // 1..3
  struct Scalars { StepCoef k; float nz; UniPcStep u; };
  __device__ __forceinline__ Scalars scalars(const StepParams& p) const {
    return {p.table[*p.t_index], (*p.t_prev != 0) ? 1.0f : 0.0f, *u};
  }
  template <typename Load>
  __device__ __forceinline__ void operator()(const StepParams& p, const Scalars& s, const Quad& q, Load&& load) const {
    auto mul = [](float a, float b) { return __fmul_rn(a, b); };
    auto add = [](float a, float b) { return __fadd_rn(a, b); };
    const UniPcStep& u = s.u;
    float h[3][4] = {}, base[4];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      if (j < depth) {
        const float4 t = *reinterpret_cast<const float4*>(arena + j * plane + q.i);
        h[j][0] = t.x; h[j][1] = t.y; h[j][2] = t.z; h[j][3] = t.w;
      }
    }
    {
      const float4 t = *reinterpret_cast<const float4*>(arena + 3 * plane + q.i);
      base[0] = t.x; base[1] = t.y; base[2] = t.z; base[3] = t.w;
    }
    float xt[4], x0[4], xc[4], xo[4];
    load(xt, x0);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float d = guide_x0(p, s.nz, q.n, q.c, q.pix + e, x0[e]);
      x0[e] = d;
      float v = xt[e];
      if (u.corr_order >= 1) {
        v = add(mul(u.a, base[e]), mul(u.v[0], d));
#pragma unroll
        for (int j = 0; j < 3; ++j)
          if (j < u.corr_order) v = add(v, mul(u.v[j + 1], h[j][e]));
      }
      xc[e] = v;
      float o = add(mul(u.c, v), mul(u.w[0], d));
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (j + 1 < u.order) o = add(o, mul(u.w[j + 1], h[j][e]));
      xo[e] = o;
    }
    stg_f4(p.x_prev + q.i, make_float4(xo[0], xo[1], xo[2], xo[3]));
    if (p.pred_x0) stg_f4(p.pred_x0 + q.i, make_float4(x0[0], x0[1], x0[2], x0[3]));
    if (corrected) stg_f4(corrected + q.i, make_float4(xc[0], xc[1], xc[2], xc[3]));
    stg_f4(arena + 3 * plane + q.i, make_float4(xc[0], xc[1], xc[2], xc[3]));
#pragma unroll
    for (int j = 2; j >= 1; --j)
      if (j < depth) stg_f4(arena + j * plane + q.i, make_float4(h[j - 1][0], h[j - 1][1], h[j - 1][2], h[j - 1][3]));
    stg_f4(arena + q.i, make_float4(x0[0], x0[1], x0[2], x0[3]));
  }
};

// x_0 of a quad into a [N,C,H,W] buffer.  x0 may be the eps buffer of an EpsRows source (rows [0,N)): each element is read
// before it is overwritten, by the same thread, so neither pointer is __restrict__.
struct StoreX0 {
  float* x0;
  struct Scalars { StepCoef k; };
  __device__ __forceinline__ static Scalars scalars(const StepParams& p) { return {p.table[*p.t_index]}; }
  template <typename Load>
  __device__ __forceinline__ void operator()(const StepParams&, const Scalars&, const Quad& q, Load&& load) const {
    float xt[4], v[4];
    load(xt, v);
    stg_f4(x0 + q.i, make_float4(v[0], v[1], v[2], v[3]));
  }
};

// The first pass of an APG step (a source reading ApgInputs): D_c, m = (D_c - D_u) + beta * m_prev and the PAG term of a
// quad into the planes of a.  On a step the device flag leaves unguided only D_c is written and m_prev stays as it was.
struct ApgStore {
  ApgParams a;
  using Reader = ApgInputs;
  struct Scalars { StepCoef k; int guided; };
  __device__ __forceinline__ static Scalars scalars(const StepParams& p) { return {p.table[*p.t_index], step_cfg(p) & 3}; }
  template <typename Load>
  __device__ __forceinline__ void operator()(const StepParams& p, const Scalars& s, const Quad& q, Load&& load) const {
    float xt[4], in[3][4];
    load(xt, in);
    stg_f4(a.dc + q.i, make_float4(in[0][0], in[0][1], in[0][2], in[0][3]));
    if (!s.guided) return;
    float mp[4] = {0.f, 0.f, 0.f, 0.f}, m[4];
    if (a.beta != 0.0f) {
      const float4 t = *reinterpret_cast<const float4*>(a.m + q.i);
      mp[0] = t.x; mp[1] = t.y; mp[2] = t.z; mp[3] = t.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) m[j] = apg_momentum(in[1][j], a.beta, mp[j]);
    stg_f4(a.m + q.i, make_float4(m[0], m[1], m[2], m[3]));
    if (p.pag) stg_f4(a.pag + q.i, make_float4(in[2][0], in[2][1], in[2][2], in[2][3]));
  }
};

// x_0 of an APG step from the planes of the first pass and the scalars of apg_reduce_kernel: D = D_c + s c (m - k D_c), plus
// the PAG term (cfg & kPagBit), clipped when p.clip is set; D_c alone (then clipped) on a step the device flag leaves
// unguided (cfg 0), which is the unguided step's x_0 bit for bit.  One quad per unit.
struct ApgX0 {
  ApgParams a;
  __host__ __device__ size_t units(const StepParams& p) const { return static_cast<size_t>(p.N) * p.C * p.HW / 4; }
  template <typename F>
  __device__ __forceinline__ void quads(const StepParams& p, const StepCoef&, int cfg, size_t u, F&& f) const {
    const Quad q = flat_quad(p, u);
    f(q, [&](float (&xt)[4], float (&x0)[4]) {
      const float4 d = ldg_f4(a.dc + q.i);
      const float dc[4] = {d.x, d.y, d.z, d.w};
      float dv[4] = {dc[0], dc[1], dc[2], dc[3]};
      if (cfg & 3) {
        const float sc = a.scal[2 * q.n], sck = a.scal[2 * q.n + 1];
        const float4 m = ldg_f4(a.m + q.i);
        const float mv[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) dv[j] = apg_guide(dc[j], mv[j], sc, sck);
        if (cfg & kPagBit) {
          const float4 g = ldg_f4(a.pag + q.i);
          dv[0] = __fadd_rn(dv[0], g.x); dv[1] = __fadd_rn(dv[1], g.y);
          dv[2] = __fadd_rn(dv[2], g.z); dv[3] = __fadd_rn(dv[3], g.w);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        xt[j] = p.x_t[q.i + j];
        x0[j] = p.clip ? fminf(fmaxf(dv[j], -1.0f), 1.0f) : dv[j];
      }
    });
  }
};

// kPag: the instantiation for steps with perturbed-attention guidance (p.pag = 1); the others mask kPagBit off at compile time.
// The APG first pass (Sink = ApgStore) has its source read ApgInputs instead of the guided x_0.
template <typename Src, typename Sink, bool kPag>
__global__ void __launch_bounds__(256) step_kernel(const StepParams p, const Src src, const Sink sink) {
  const typename Sink::Scalars s = sink.scalars(p);
  const int cfg = kPag ? step_cfg(p) : (step_cfg(p) & 3);
  const size_t units = src.units(p);
  for (size_t u = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; u < units; u += static_cast<size_t>(gridDim.x) * blockDim.x) {
    if constexpr (std::is_same_v<Sink, ApgStore>)
      src.template quads<ApgInputs>(p, s.k, cfg, u, [&](const Quad& q, auto&& load) { sink(p, s, q, load); });
    else
      src.quads(p, s.k, cfg, u, [&](const Quad& q, auto&& load) { sink(p, s, q, load); });
  }
}

// The two scalars of APG for every sample n (one block per sample) from the first pass's planes D_c and m over its M elements:
// |m|^2, <m, D_c> and |D_c|^2 in double, each thread over elements threadIdx.x + j * kApgThreads in order, then a fixed
// tree over the block, so the sums depend on the sample's own elements only.  c = min(1, r / |m|) (1 for r = 0 or m = 0),
// k = (1 - eta) <m, D_c> / max(|D_c|^2, tiny); scal[n] = {fp32(s) * fp32(c), fp32(s * fp32(c) * k)}.  guided != nullptr
// and 0: the step is unguided and nothing is written.
constexpr int kApgThreads = 512;
__global__ void __launch_bounds__(kApgThreads) apg_reduce_kernel(const float* __restrict__ dc, const float* __restrict__ m, int M,
                                                                 float s, double eta, double r, const int* guided,
                                                                 float* __restrict__ scal) {
  if (guided != nullptr && *guided == 0) return;
  __shared__ double part[3][kApgThreads / 32];
  const size_t base = static_cast<size_t>(blockIdx.x) * M;
  double mm = 0.0, md = 0.0, dd = 0.0;
  for (int i = threadIdx.x; i < M; i += kApgThreads) {
    const double mv = m[base + i], dv = dc[base + i];
    mm = __fma_rn(mv, mv, mm);
    md = __fma_rn(mv, dv, md);
    dd = __fma_rn(dv, dv, dd);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mm = __dadd_rn(mm, __shfl_xor_sync(0xFFFFFFFFu, mm, o));
    md = __dadd_rn(md, __shfl_xor_sync(0xFFFFFFFFu, md, o));
    dd = __dadd_rn(dd, __shfl_xor_sync(0xFFFFFFFFu, dd, o));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { part[0][warp] = mm; part[1][warp] = md; part[2][warp] = dd; }
  __syncthreads();
  if (threadIdx.x == 0) {
    mm = md = dd = 0.0;
    for (int w = 0; w < kApgThreads / 32; ++w) {
      mm = __dadd_rn(mm, part[0][w]);
      md = __dadd_rn(md, part[1][w]);
      dd = __dadd_rn(dd, part[2][w]);
    }
    const double nm = sqrt(mm);
    const float c = (r > 0.0 && nm > 0.0) ? static_cast<float>(fmin(1.0, r / nm)) : 1.0f;
    const double k = (1.0 - eta) * md / fmax(dd, 2.2250738585072014e-308);
    scal[2 * blockIdx.x] = __fmul_rn(s, c);
    scal[2 * blockIdx.x + 1] = static_cast<float>(static_cast<double>(s) * c * k);
  }
}

// The element passes of ivid_op_apg over [N][M]: m = (d_c - d_u) + beta * m_prev in place, then out = apg_guide
__global__ void __launch_bounds__(256) apg_momentum_kernel(const float* __restrict__ dc, const float* __restrict__ du, float* m,
                                                           float beta, size_t total) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    m[i] = apg_momentum(__fsub_rn(dc[i], du[i]), beta, m[i]);
}
__global__ void __launch_bounds__(256) apg_apply_kernel(const float* __restrict__ dc, const float* __restrict__ m,
                                                        const float* __restrict__ scal, float* __restrict__ out, size_t M,
                                                        size_t total) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t n = i / M;
    out[i] = apg_guide(dc[i], m[i], scal[2 * n], scal[2 * n + 1]);
  }
}

// ----------------------------------------------------------------------------------------------
// Dynamic thresholding of x_0 (Saharia et al. 2022, arXiv:2205.11487, sec. 2.3), per sample n over its M = C*H*W elements:
//   q = the ratio-quantile of |x_0| with linear interpolation (v_k + f * (v_{k+1} - v_k), pos = ratio * (M - 1) = k + f, in
//       double, rounded once to fp32), s = min(max(q, 1), s_max), x_0 <- clamp(x_0, -s, s) / s.
// A step in this mode runs three kernels: step_kernel<Src, StoreX0> (x_0 before thresholding into a [N,C,H,W] buffer, from
// HeadTaps on the fused route and EpsRows on the separate one), threshold_select_kernel (s of every sample) and
// step_kernel<ThresholdedX0, Update<kind>>.  Both routes share the last two, so they agree bit for bit.
// ----------------------------------------------------------------------------------------------

// Exact per-sample selection: one block per sample n of x [N][M] radix-selects the order statistic v_k of |x| over the fp32 bit
// patterns (ordered like unsigned integers for non-negative floats) in three digit passes, bits 31..21, 20..10 and 9..0, each a
// shared-memory histogram of the elements that share the digits found so far.  Integer counts make s exact and deterministic,
// and a sample's s depends on its own elements only.  v_{k+1} comes from the last pass: v_k again while its bin holds more
// elements, else the next non-empty bin, else the smallest element above the last pass's group.
constexpr int kSelectThreads = 1024;
// exclusive prefix sum of v over the block (kSelectThreads threads)
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* warp_sums) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, w, o);
      if (lane >= o) w += y;
    }
    warp_sums[lane] = w;
  }
  __syncthreads();
  const uint32_t r = x - v + (warp > 0 ? warp_sums[warp - 1] : 0u);
  __syncthreads();
  return r;
}
__global__ void __launch_bounds__(kSelectThreads) threshold_select_kernel(const float* __restrict__ x, int M, double ratio,
                                                                          float s_max, float* __restrict__ s_out) {
  __shared__ uint32_t hist[2048];
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t sh_bin, sh_rank, sh_next, sh_above;
  const float* xs = x + static_cast<size_t>(blockIdx.x) * M;
  const double pos = __dmul_rn(ratio, static_cast<double>(M - 1));
  const double kd = floor(pos);
  const double f = __dsub_rn(pos, kd);
  uint32_t rank = static_cast<uint32_t>(kd);   // rank of v_k among the elements that share the digits found so far
  uint32_t prefix = 0;                         // those digits
  uint32_t above = 0xFFFFFFFFu;                // last pass: the smallest key above its group (|x| < 2^31: never a key)
  if (threadIdx.x == 0) { sh_next = 0xFFFFFFFFu; sh_above = 0xFFFFFFFFu; }
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
    const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
    const int bits = pass == 2 ? 10 : 11;
    for (int b = threadIdx.x; b < 2048; b += kSelectThreads) hist[b] = 0u;
    __syncthreads();
    for (int i = threadIdx.x; i < M; i += kSelectThreads) {
      const uint32_t key = __float_as_uint(fabsf(xs[i]));
      if (pass == 0) {
        atomicAdd(&hist[key >> shift], 1u);
      } else {
        const uint32_t hi = key >> (shift + bits);
        if (hi == prefix) atomicAdd(&hist[(key >> shift) & ((1u << bits) - 1u)], 1u);
        else if (pass == 2 && hi > prefix) above = min(above, key);
      }
    }
    __syncthreads();
    // the bin that holds rank: thread t owns bins 2t and 2t + 1
    const uint32_t c0 = hist[2 * threadIdx.x], c1 = hist[2 * threadIdx.x + 1];
    const uint32_t before = block_exclusive_scan(c0 + c1, warp_sums);
    if (rank >= before && rank < before + c0 + c1) {
      const bool lo = rank < before + c0;
      sh_bin = 2 * threadIdx.x + (lo ? 0u : 1u);
      sh_rank = rank - before - (lo ? 0u : c0);
    }
    __syncthreads();
    rank = sh_rank;
    prefix = (prefix << bits) | sh_bin;
  }
  const uint32_t bin = prefix & 0x3FFu;
  for (int b = threadIdx.x; b < 1024; b += kSelectThreads)
    if (b > static_cast<int>(bin) && hist[b] != 0u) atomicMin(&sh_next, static_cast<uint32_t>(b));
  above = __reduce_min_sync(0xFFFFFFFFu, above);
  if ((threadIdx.x & 31) == 0) atomicMin(&sh_above, above);
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t next = prefix;                                          // k = M - 1: v_{min(k+1, M-1)} = v_k
    if (rank + 1 < hist[bin]) next = prefix;
    else if (sh_next != 0xFFFFFFFFu) next = (prefix & ~0x3FFu) | sh_next;
    else if (sh_above != 0xFFFFFFFFu) next = sh_above;
    const double vk = __uint_as_float(prefix), vk1 = __uint_as_float(next);
    const float q = __double2float_rn(__dadd_rn(vk, __dmul_rn(f, __dsub_rn(vk1, vk))));
    s_out[blockIdx.x] = fminf(fmaxf(q, 1.0f), s_max);
  }
}

// the clamp / scale alone (ivid_op_dynamic_threshold): out = threshold_x0(x, s[i / M]) over x [N][M]
__global__ void __launch_bounds__(256) threshold_apply_kernel(const float* __restrict__ x, const float* __restrict__ s_n, float* __restrict__ out,
                                                              size_t M, size_t total) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    out[i] = threshold_x0(x[i], s_n[i / M]);
}

// ----------------------------------------------------------------------------------------------
// Conditional-model input assembly, fused with the NCHW fp32 -> NHWC fp16(64 ch) packing.
// ----------------------------------------------------------------------------------------------
struct CondPackParams {
  const float* x;         // [Nx,4,H,W]
  const float* y;         // inpaint: [Nx,4,H,W] warped RGBD;  superres: [Nx,4,H/s,W/s] low-res RGBD
  const float* mask;      // inpaint [Nx,1,H,W]
  const float* mask_rgb;  // inpaint [Nx,1,H,W] or nullptr (then mask is used and no mask_rgb channel is emitted)
  const float* noise;     // inpaint: injected [Nx,4,H,W] (rgb noise 3 + depth noise 1) or nullptr -> Philox
  __half* out;            // [N,H,W,64]
  int N, Nx, H, W;
  int kind;               // 1 = InpaintCFG, 2 = SuperResCFG
  int scale;              // superres: integer upsampling factor s
  float inv_scale;        // superres: (float)(1.0 / s), the source-index scale of ATen's upsample_bilinear2d(scale_factor=s)
  uint64_t seed;
  uint32_t stream;
  const int* stream_dev;
};

__global__ void __launch_bounds__(256) cond_pack_kernel(const CondPackParams p) {
  // phase 1: one thread per pixel assembles the Cin (<= 16) fp32 input channels into shared memory;
  // phase 2: the block writes the 64 fp16 operand channels (two-term split hi | lo | hi, see pack_input_kernel) with
  //          16-byte coalesced stores, one thread per (pixel, 8-channel group).
  __shared__ float s_ch[256][17];
  const int HW = p.H * p.W;
  const size_t total = static_cast<size_t>(p.N) * HW;
  const uint32_t stream = p.stream + (p.stream_dev ? static_cast<uint32_t>(*p.stream_dev) : 0u);
  const int Cin = p.kind == 1 ? (p.mask_rgb ? 10 : 9) : 8;
  for (size_t base = blockIdx.x * static_cast<size_t>(blockDim.x); base < total; base += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t idx = base + threadIdx.x;
    if (idx < total) {
      const int n = static_cast<int>(idx / HW) % p.Nx;
      const int pix = static_cast<int>(idx % HW);
      float ch[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) ch[j] = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) ch[c] = p.x[(static_cast<size_t>(n) * 4 + c) * HW + pix];
      if (p.kind == 1) {
        const float m = p.mask[static_cast<size_t>(n) * HW + pix];
        const float mr = p.mask_rgb ? p.mask_rgb[static_cast<size_t>(n) * HW + pix] : m;
        float z[4];
        if (p.noise != nullptr) {
#pragma unroll
          for (int c = 0; c < 4; ++c) z[c] = p.noise[(static_cast<size_t>(n) * 4 + c) * HW + pix];
        } else {
          const float4 t = philox_normal4(p.seed, stream, static_cast<uint32_t>(static_cast<size_t>(n) * HW + pix));
          z[0] = t.x; z[1] = t.y; z[2] = t.z; z[3] = t.w;
        }
        int o = 4;
        if (p.mask_rgb) ch[o++] = mr;
#pragma unroll
        for (int c = 0; c < 3; ++c)
          ch[o++] = p.y[(static_cast<size_t>(n) * 4 + c) * HW + pix] * mr + z[c] * (1.0f - mr);
        ch[o++] = p.y[(static_cast<size_t>(n) * 4 + 3) * HW + pix] * m + z[3] * (1.0f - m);
        ch[o++] = m;
      } else {
        // bilinear s-x upsample, align_corners=False: src = (dst + 0.5) * (1/s) - 0.5, clamped at 0 (ATen upsample_bilinear2d
        // with scale_factor=s); for s = 2 the factor is exactly 0.5
        const int h = pix / p.W, w = pix % p.W;
        const int Hs = p.H / p.scale, Ws = p.W / p.scale;
        float sy = (h + 0.5f) * p.inv_scale - 0.5f; if (sy < 0.f) sy = 0.f;
        float sx = (w + 0.5f) * p.inv_scale - 0.5f; if (sx < 0.f) sx = 0.f;
        const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
        const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
        const float ly = sy - y0, lx = sx - x0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float* s = p.y + (static_cast<size_t>(n) * 4 + c) * Hs * Ws;
          const float v = (1.f - ly) * ((1.f - lx) * s[y0 * Ws + x0] + lx * s[y0 * Ws + x1]) +
                          ly * ((1.f - lx) * s[y1 * Ws + x0] + lx * s[y1 * Ws + x1]);
          ch[4 + c] = v;
        }
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) s_ch[threadIdx.x][j] = ch[j];
    }
    __syncthreads();
    const int live = static_cast<int>(min(static_cast<size_t>(256), total - base));
    for (int it = threadIdx.x; it < live * 8; it += 256) {
      const int px = it >> 3, g = it & 7;
      uint32_t w4[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        __half e[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int oc = g * 8 + 2 * k + q;
          const int seg = oc / Cin;
          e[q] = seg < 3 ? split_term(s_ch[px][oc - seg * Cin], seg) : __float2half_rn(0.f);
        }
        const __half2 h2 = __halves2half2(e[0], e[1]);
        w4[k] = *reinterpret_cast<const uint32_t*>(&h2);
      }
      *reinterpret_cast<uint4*>(p.out + (base + px) * 64 + g * 8) = make_uint4(w4[0], w4[1], w4[2], w4[3]);
    }
    __syncthreads();
  }
}

}  // namespace ivid
