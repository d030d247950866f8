// HBM-bound element-wise kernels of the ADM UNet hot path (NHWC fp32 residual stream -> fp16 MMA operands).
//
//   gn_stats_kernel  : per-(sample, channel) sum / sum-of-squares of an fp32 NHWC tensor (double accumulators).
//                      GroupNorm32 statistics (reference adm.py:36-41) are later formed per group from these, which
//                      is what makes GroupNorm over a *virtual* channel concat (groups straddling the seam,
//                      adm.py:563 + :158) free of any concat copy.
//                      Only used below 32 pixels per sample and after the pooling / nearest resampling layers: everywhere
//                      else the producing conv's epilogue accumulates the statistics.  Each thread sums its pixels in
//                      fp32, at most ceil(min(HW, 256) / rows) of them (rows = 256 / min(C/4, 256)); the rest is fp64.
//   gn_prologue      : (device function, per block) per-(sample, channel) affine y = x*A + B that folds mean/rstd,
//                      gamma/beta and the FiLM scale/shift  h = GN(h)*(1+scale)+shift  (adm.py:216-217).
//   gn_apply_h16_kernel: y = [SiLU](x*A+B), fp16 NHWC sources (hidden tensor, fp16 copies of block outputs, virtual
//                      concat of two) -> fp16 NHWC conv operand; the bulk of the traffic.
//   gn_apply_kernel  : generic variant: fp32 sources, the ResBlock's nearest-2x upsample / 2x2 average pool
//                      (adm.py:203-208), optional raw fp16 copy (operand of the 1x1 skip conv) and / or resampled fp32
//                      copy (identity skip of up/down blocks).
//   pack_input_kernel: NCHW fp32 network input -> NHWC fp16 padded to 64 channels (adm.py:557, x.type(dtype)).
#pragma once
#include "common.cuh"

namespace ivid {

// ----------------------------------------------------------------------------------------------
// per-channel statistics.  grid = (ceil(HW / PIX_PER_BLOCK), N), block = 256.
// ----------------------------------------------------------------------------------------------
constexpr int kStatsPixPerBlock = 256;

__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, double* __restrict__ stats,
                                                       int HW, int C) {
  // thread layout: tx over C/4 float4 columns, ty over pixel rows
  __shared__ float sred[256 * 8];   // [rows][cols][8] partials -> reduced over rows
  const int n = blockIdx.y;
  const int c4 = C >> 2;
  const int cols = c4 < 256 ? c4 : 256;        // threads across channels
  const int rows = 256 / cols;                 // pixel rows handled concurrently
  const int tx = threadIdx.x % cols;
  const int ty = threadIdx.x / cols;
  const int p0 = blockIdx.x * kStatsPixPerBlock;
  const int p1 = min(p0 + kStatsPixPerBlock, HW);
  const float* base = x + (static_cast<size_t>(n) * HW) * C;
  // Every thread runs the same ceil(c4 / cols) rounds, so the whole block reaches each barrier.  When C/4 > 256 is not a
  // multiple of 256 the last round leaves columns cc >= c4 idle: they load nothing and store nothing to the statistics.
  for (int cc0 = 0; cc0 < c4; cc0 += cols) {
    const int cc = cc0 + tx;
    const bool live = cc < c4;
    float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
    if (ty < rows && live) {
      for (int p = p0 + ty; p < p1; p += rows) {
        const float4 v = ldg_f4(base + static_cast<size_t>(p) * C + cc * 4);
        s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
        q[0] += v.x * v.x; q[1] += v.y * v.y; q[2] += v.z * v.z; q[3] += v.w * v.w;
      }
    }
    // reduce over ty through shared memory (rows <= 8 for C >= 128)
    float* sm = sred;   // [rows][cols][8]
    if (ty < rows) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        sm[(ty * cols + tx) * 8 + j] = s[j];
        sm[(ty * cols + tx) * 8 + 4 + j] = q[j];
      }
    }
    __syncthreads();
    if (ty == 0 && live) {
      double ds[4], dq[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { ds[j] = 0.0; dq[j] = 0.0; }
      for (int r = 0; r < rows; ++r) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          ds[j] += static_cast<double>(sm[(r * cols + tx) * 8 + j]);
          dq[j] += static_cast<double>(sm[(r * cols + tx) * 8 + 4 + j]);
        }
      }
      double* o = stats + (static_cast<size_t>(n) * C + cc * 4) * 2;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        atomicAdd(o + 2 * j, ds[j]);
        atomicAdd(o + 2 * j + 1, dq[j]);
      }
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------------------------
// GroupNorm apply (+FiLM, +SiLU, +resample).  grid = (pixel chunks, N), block = 256.
// Prologue (per block): group mean / rstd of sample n from the per-channel statistics of up to two sources (virtual
// concat: channels [0,C0) from stats0, [C0,C0+C1) from stats1), folded with gamma/beta and the FiLM scale/shift into a
// per-channel affine kept in shared memory:
//   A[c] = rstd*gamma*(1+scale),  B[c] = (beta - mean*rstd*gamma)*(1+scale) + shift
//   film: [N][film_ld] table; scale = film[n][film_off + c], shift = film[n][film_off + C + c]  (torch.chunk(emb_out, 2)).
// Body: one work item = 8 channels of one OUTPUT pixel.
//   mode 0: same resolution; 1: nearest 2x upsample (Ho = 2H); 2: 2x2 average pool (Ho = H/2)
// ----------------------------------------------------------------------------------------------
struct GnApplyParams {
  const float* x0; const float* x1;     // fp32 NHWC sources (virtual concat along C); x1 may be null (C1 = 0)
  const __half* x0h; const __half* x1h; // when x0h is non-null the sources are fp16 NHWC (hidden tensor / fp16 copies)
  int C0, C1;
  int N, H, W;                          // INPUT spatial size
  int mode;                             // 0 same, 1 up, 2 down
  int silu;                             // 0 none, 1 SiLU (silu_f)
  const double* stats0; const double* stats1;   // [N][C0][2], [N][C1][2] (sum, sum of squares over H*W)
  int groups; double inv_count; float eps;
  const float* gamma; const float* beta;
  const float* film; int film_ld, film_off;
  int film_add;                         // 1: use_scale_shift_norm=False (adm.py:219-221): y = GN(x + e[n][c]) with e = film[n][film_off + c]
                                        //    added BEFORE the norm; the group moments of x + e follow from the per-channel ones
  int pix_per_block;
  __half* out_act;                      // fp16 [N][Ho][Wo][C]
  __half* out_lo;                       // optional (same-resolution fp16-source path only): fp16(y - float(fp16(y))), the low half
                                        // of a two-term split of the activation (operand of the split-precision output conv)
  __half* out_raw16;                    // optional fp16 raw copy (same-resolution only) [N][H][W][C]
  float* out_raw32;                     // optional fp32 raw (resampled) [N][Ho][Wo][C]
  uint8_t* out_act8;                    // the kF8 kernels write the activation here instead, as e4m3 [N][Ho][Wo][C]
};

// 8 activations of one work item as the operand the next conv reads: fp16 (16 bytes) or, kF8, e4m3 (8 bytes, satfinite)
template <bool kF8> struct Act8 { using T = uint4; };
template <> struct Act8<true> { using T = uint2; };
template <bool kF8>
__device__ __forceinline__ typename Act8<kF8>::T pack_act8(const float (&a)[8]) {
  if constexpr (kF8) {
    uint2 pk;
    pk.x = pack_e4m3x2(a[0], a[1]) | (static_cast<uint32_t>(pack_e4m3x2(a[2], a[3])) << 16);
    pk.y = pack_e4m3x2(a[4], a[5]) | (static_cast<uint32_t>(pack_e4m3x2(a[6], a[7])) << 16);
    return pk;
  } else {
    uint4 pk;
    pk.x = pack_h2(a[0], a[1]); pk.y = pack_h2(a[2], a[3]);
    pk.z = pack_h2(a[4], a[5]); pk.w = pack_h2(a[6], a[7]);
    return pk;
  }
}
// element offset o of the activation output
template <bool kF8>
__device__ __forceinline__ void store_act8(const GnApplyParams& p, size_t o, const typename Act8<kF8>::T& v) {
  if constexpr (kF8) *reinterpret_cast<uint2*>(p.out_act8 + o) = v;
  else *reinterpret_cast<uint4*>(p.out_act + o) = v;
}

__device__ __forceinline__ void load8(const GnApplyParams& p, int n, int h, int w, int c, float (&v)[8]) {
  if (p.x0h != nullptr) {
    const __half* hs; int hc, hl;
    if (c < p.C0) { hs = p.x0h; hc = c; hl = p.C0; } else { hs = p.x1h; hc = c - p.C0; hl = p.C1; }
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(hs + ((static_cast<size_t>(n) * p.H + h) * p.W + w) * hl + hc));
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h2[j]); v[2 * j] = f.x; v[2 * j + 1] = f.y; }
    return;
  }
  const float* src;
  int cc, ld;
  if (c < p.C0) { src = p.x0; cc = c; ld = p.C0; } else { src = p.x1; cc = c - p.C0; ld = p.C1; }
  const float* q = src + ((static_cast<size_t>(n) * p.H + h) * p.W + w) * ld + cc;
  const float4 a = ldg_f4(q), b = ldg_f4(q + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// Block -> (sample, pixel chunk)
__device__ __forceinline__ void gn_block_pos(const GnApplyParams&, int& n, int& bx) {
  n = static_cast<int>(blockIdx.y);
  bx = static_cast<int>(blockIdx.x);
}

// statistics -> per-channel affine (see above) for sample blockIdx.y, left in shared memory for the whole block
__device__ __forceinline__ void gn_prologue(const GnApplyParams& p, float* s_ab, float* s_mean, float* s_rstd) {
  const int C = p.C0 + p.C1;
  int n, bx_unused;
  gn_block_pos(p, n, bx_unused);
  const int cpg = C / p.groups;
  if ((cpg & (cpg - 1)) == 0 && cpg <= 32 && C % 32 == 0 && C <= 4 * 256 && blockDim.x == 256) {
    // fast path (power-of-two group width): thread = channel; every global load of the prologue (statistics and affine /
    // FiLM parameters) is issued up front, the group sums are formed by shuffles, and there is a single barrier.
    // C % 32 == 0 keeps the full-warp shuffles on whole warps; other widths (e.g. 40 = 8 groups of 5) take the loop below
    constexpr int PF = 4;
    double2 st[PF];
    float pg[PF], pb[PF], psc[PF], psh[PF];
#pragma unroll
    for (int i = 0; i < PF; ++i) {
      const int c = threadIdx.x + i * 256;
      if (c < C) {
        const double* sp = (c < p.C0) ? p.stats0 + (static_cast<size_t>(n) * p.C0 + c) * 2
                                      : p.stats1 + (static_cast<size_t>(n) * p.C1 + (c - p.C0)) * 2;
        st[i] = *reinterpret_cast<const double2*>(sp);
        pg[i] = p.gamma[c];
        pb[i] = p.beta[c];
        if (p.film != nullptr) {
          psc[i] = p.film[static_cast<size_t>(n) * p.film_ld + p.film_off + c];
          psh[i] = p.film_add ? 0.f : p.film[static_cast<size_t>(n) * p.film_ld + p.film_off + C + c];
          if (p.film_add) {
            // sum(x + e) = S + HW e ; sum((x + e)^2) = Q + 2 e S + HW e^2   (HW = 1 / inv_count)
            const double e = static_cast<double>(psc[i]), hw = 1.0 / p.inv_count;
            const double S = st[i].x;
            st[i].x = S + hw * e;
            st[i].y = st[i].y + 2.0 * e * S + hw * e * e;
          }
        }
      }
    }
    const double cnt_inv = p.inv_count / cpg;
#pragma unroll
    for (int i = 0; i < PF; ++i) {
      const int c = threadIdx.x + i * 256;
      if (c < C) {            // C % 32 == 0: whole warps take the branch together
        double sm = st[i].x, q = st[i].y;
        for (int off = 1; off < cpg; off <<= 1) {
          sm += __shfl_xor_sync(0xffffffffu, sm, off);
          q += __shfl_xor_sync(0xffffffffu, q, off);
        }
        const double mean = sm * cnt_inv;
        double var = q * cnt_inv - mean * mean;
        if (var < 0.0) var = 0.0;
        const float rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(p.eps)));
        const float a0 = rstd * pg[i];
        const float b0 = pb[i] - static_cast<float>(mean) * a0;
        float av = a0, bv = b0;
        if (p.film != nullptr && p.film_add) {
          bv = fmaf(psc[i], a0, b0);          // (x + e - mean) * rstd * gamma + beta
        } else if (p.film != nullptr) {
          const float sc = 1.0f + psc[i];
          av = a0 * sc;
          bv = b0 * sc + psh[i];
        }
        s_ab[(c & 7) * (C >> 3) + (c >> 3)] = av;
        s_ab[C + (c & 7) * (C >> 3) + (c >> 3)] = bv;
      }
    }
    __syncthreads();
    return;
  }
  for (int g = threadIdx.x; g < p.groups; g += blockDim.x) {
    double s = 0.0, q = 0.0;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
      const double* st = (c < p.C0) ? p.stats0 + (static_cast<size_t>(n) * p.C0 + c) * 2
                                    : p.stats1 + (static_cast<size_t>(n) * p.C1 + (c - p.C0)) * 2;
      double sc = st[0], qc = st[1];
      if (p.film != nullptr && p.film_add) {
        const double e = static_cast<double>(p.film[static_cast<size_t>(n) * p.film_ld + p.film_off + c]), hw = 1.0 / p.inv_count;
        qc = qc + 2.0 * e * sc + hw * e * e;
        sc = sc + hw * e;
      }
      s += sc;
      q += qc;
    }
    const double cnt_inv = p.inv_count / cpg;
    const double mean = s * cnt_inv;
    double var = q * cnt_inv - mean * mean;
    if (var < 0.0) var = 0.0;
    s_mean[g] = static_cast<float>(mean);
    s_rstd[g] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(p.eps)));
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float a0 = s_rstd[g] * p.gamma[c];
    const float b0 = p.beta[c] - s_mean[g] * a0;
    float a = a0, b = b0;
    if (p.film != nullptr && p.film_add) {
      b = fmaf(p.film[static_cast<size_t>(n) * p.film_ld + p.film_off + c], a0, b0);
    } else if (p.film != nullptr) {
      const float sc = 1.0f + p.film[static_cast<size_t>(n) * p.film_ld + p.film_off + c];
      const float sh = p.film[static_cast<size_t>(n) * p.film_ld + p.film_off + C + c];
      a = a0 * sc;
      b = b0 * sc + sh;
    }
    s_ab[(c & 7) * (C >> 3) + (c >> 3)] = a;
    s_ab[C + (c & 7) * (C >> 3) + (c >> 3)] = b;
  }
  __syncthreads();

}

template <bool kF8 = false>
__global__ void __launch_bounds__(256, 3) gn_apply_kernel(const GnApplyParams p) {
  extern __shared__ float s_ab[];        // A then B, each stored [c % 8][c / 8] so a warp's reads are conflict-free
  __shared__ float s_mean[64], s_rstd[64];
  gn_prologue(p, s_ab, s_mean, s_rstd);
  const int C = p.C0 + p.C1;
  int n, bx;
  gn_block_pos(p, n, bx);
  const int c8 = C >> 3;
  const int Ho = p.mode == 1 ? p.H * 2 : (p.mode == 2 ? p.H / 2 : p.H);
  const int Wo = p.mode == 1 ? p.W * 2 : (p.mode == 2 ? p.W / 2 : p.W);
  const int pix0 = bx * p.pix_per_block;
  if (p.mode == 1) {
    // nearest-2x upsample, source-centric (pix_per_block counts SOURCE pixels): each source item is loaded and activated
    // once and written to its 2x2 output pixels (fp16 operand + the resampled fp32 identity skip)
    const int npix_s = min(p.pix_per_block, p.H * p.W - pix0);
    const int items_s = npix_s * c8;
    constexpr int U = 4;
    auto emit = [&](int it, const float (&raw)[8]) {
      const int cg = it % c8;
      const int pix = pix0 + it / c8;
      const int hs = pix / p.W, ws = pix - hs * p.W;
      float act[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float y = fmaf(raw[j], s_ab[j * c8 + cg], s_ab[C + j * c8 + cg]);
        if (p.silu) y = silu_f(y);
        act[j] = y;
      }
      const auto pk = pack_act8<kF8>(act);
      const float4 r0 = make_float4(raw[0], raw[1], raw[2], raw[3]), r1 = make_float4(raw[4], raw[5], raw[6], raw[7]);
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const size_t o = ((static_cast<size_t>(n) * Ho + 2 * hs + dy) * Wo + 2 * ws + dx) * C + cg * 8;
          store_act8<kF8>(p, o, pk);
          if (p.out_raw32 != nullptr) { stg_f4(p.out_raw32 + o, r0); stg_f4(p.out_raw32 + o + 4, r1); }
        }
    };
    int it0 = threadIdx.x;
    for (; it0 + (U - 1) * 256 < items_s; it0 += U * 256) {
      float raw[U][8];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int it = it0 + u * 256;
        const int pix = pix0 + it / c8;
        load8(p, n, pix / p.W, pix % p.W, (it % c8) * 8, raw[u]);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) emit(it0 + u * 256, raw[u]);
    }
    for (int it = it0; it < items_s; it += 256) {
      float raw[8];
      const int pix = pix0 + it / c8;
      load8(p, n, pix / p.W, pix % p.W, (it % c8) * 8, raw);
      emit(it, raw);
    }
    return;
  }
  const int npix = min(p.pix_per_block, Ho * Wo - pix0);
  const int items = npix * c8;
  int it0 = threadIdx.x;
  if (p.mode == 0) {
    // same-resolution fast path (the bulk of the traffic): 4 work items per thread per trip, all 8 x 16-byte loads issued
    // before any is consumed, so a block keeps ~32 KB of reads in flight
    constexpr int U = 4;
    for (; it0 + (U - 1) * 256 < items; it0 += U * 256) {
      float raw[U][8];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int it = it0 + u * 256;
        const int pix = pix0 + it / c8;
        load8(p, n, pix / Wo, pix % Wo, (it % c8) * 8, raw[u]);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int it = it0 + u * 256;
        const int cg = it % c8;
        const int pix = pix0 + it / c8;
        const size_t o = (static_cast<size_t>(n) * Ho * Wo + pix) * C + cg * 8;
        float act[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float y = fmaf(raw[u][j], s_ab[j * c8 + cg], s_ab[C + j * c8 + cg]);
          if (p.silu) y = silu_f(y);
          act[j] = y;
        }
        store_act8<kF8>(p, o, pack_act8<kF8>(act));
        if (p.out_raw16 != nullptr) {
          uint4 pr;
          pr.x = pack_h2(raw[u][0], raw[u][1]); pr.y = pack_h2(raw[u][2], raw[u][3]);
          pr.z = pack_h2(raw[u][4], raw[u][5]); pr.w = pack_h2(raw[u][6], raw[u][7]);
          *reinterpret_cast<uint4*>(p.out_raw16 + o) = pr;
        }
        if (p.out_raw32 != nullptr) {
          stg_f4(p.out_raw32 + o, make_float4(raw[u][0], raw[u][1], raw[u][2], raw[u][3]));
          stg_f4(p.out_raw32 + o + 4, make_float4(raw[u][4], raw[u][5], raw[u][6], raw[u][7]));
        }
      }
    }
  }
  for (int it = it0; it < items; it += blockDim.x) {
    const int cg = it % c8;
    const int pix = pix0 + it / c8;
    const int wo = pix % Wo, ho = pix / Wo;
    const int c = cg * 8;
    float A[8], B[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { A[j] = s_ab[j * c8 + cg]; B[j] = s_ab[C + j * c8 + cg]; }
    float act[8], raw[8];
    if (p.mode == 2) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { act[j] = 0.f; raw[j] = 0.f; }
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          float v[8];
          load8(p, n, ho * 2 + dy, wo * 2 + dx, c, v);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float y = fmaf(v[j], A[j], B[j]);
            if (p.silu) y = silu_f(y);
            act[j] += y;
            raw[j] += v[j];
          }
        }
#pragma unroll
      for (int j = 0; j < 8; ++j) { act[j] *= 0.25f; raw[j] *= 0.25f; }
    } else {
      const int hi = p.mode == 1 ? (ho >> 1) : ho;
      const int wi = p.mode == 1 ? (wo >> 1) : wo;
      load8(p, n, hi, wi, c, raw);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float y = fmaf(raw[j], A[j], B[j]);
        if (p.silu) y = silu_f(y);
        act[j] = y;
      }
    }
    const size_t o = ((static_cast<size_t>(n) * Ho + ho) * Wo + wo) * C + c;
    store_act8<kF8>(p, o, pack_act8<kF8>(act));
    if (p.out_raw16 != nullptr) {
      uint4 pr;
      pr.x = pack_h2(raw[0], raw[1]); pr.y = pack_h2(raw[2], raw[3]);
      pr.z = pack_h2(raw[4], raw[5]); pr.w = pack_h2(raw[6], raw[7]);
      *reinterpret_cast<uint4*>(p.out_raw16 + o) = pr;
    }
    if (p.out_raw32 != nullptr) {
      stg_f4(p.out_raw32 + o, make_float4(raw[0], raw[1], raw[2], raw[3]));
      stg_f4(p.out_raw32 + o + 4, make_float4(raw[4], raw[5], raw[6], raw[7]));
    }
  }
}

// ----------------------------------------------------------------------------------------------
// Plain resampling layers (resblock_updown=False: Downsample2d / Upsample2d, reference adm.py:60-117)
// ----------------------------------------------------------------------------------------------
// Operand of the stride-2 3x3 convolution of Downsample2d (adm.py:111):  col[n][yo][xo][tap*C + c] = x[n][2yo+dy-1][2xo+dx-1][c]
// (zero outside the image), tap = dy*3 + dx, so that the packed 3x3 weights ([Cout][tap][C]) apply as a 1x1 GEMM over 9C channels.
__global__ void __launch_bounds__(256) im2col_s2_h16_kernel(const __half* __restrict__ x, __half* __restrict__ col, int N, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2, c8 = C >> 3;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * 9 * c8;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % c8);
    const int tap = static_cast<int>((i / c8) % 9);
    const size_t pix = i / (static_cast<size_t>(c8) * 9);
    const int xo = static_cast<int>(pix % Wo), yo = static_cast<int>((pix / Wo) % Ho);
    const int n = static_cast<int>(pix / (static_cast<size_t>(Wo) * Ho));
    const int yi = 2 * yo + tap / 3 - 1, xi = 2 * xo + tap % 3 - 1;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (yi >= 0 && yi < H && xi >= 0 && xi < W)
      v = __ldg(reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * H + yi) * W + xi) * C + cg * 8));
    *reinterpret_cast<uint4*>(col + (pix * 9 + tap) * C + cg * 8) = v;
  }
}

// Upsample2d (adm.py:89): nearest 2x of an fp16 NHWC tensor (the operand of its 3x3 conv)
__global__ void __launch_bounds__(256) upsample2x_h16_kernel(const __half* __restrict__ x, __half* __restrict__ out, int N, int H, int W, int C) {
  const int Ho = H * 2, Wo = W * 2, c8 = C >> 3;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * c8;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % c8);
    const size_t pix = i / c8;
    const int xo = static_cast<int>(pix % Wo), yo = static_cast<int>((pix / Wo) % Ho);
    const int n = static_cast<int>(pix / (static_cast<size_t>(Wo) * Ho));
    *reinterpret_cast<uint4*>(out + pix * C + cg * 8) =
        __ldg(reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * H + (yo >> 1)) * W + (xo >> 1)) * C + cg * 8));
  }
}

// conv_resample=False: AvgPool2d(2) (mode 2, adm.py:113) / nearest 2x (mode 1, adm.py:89) of an fp32 NHWC block output
// -> fp32 NHWC (+ fp16 copy for the next GroupNorm / skip conv)
__global__ void __launch_bounds__(256) resample_f32_kernel(const float* __restrict__ x, float* __restrict__ out, __half* __restrict__ out16,
                                                            int N, int H, int W, int C, int mode) {
  const int Ho = mode == 1 ? H * 2 : H / 2, Wo = mode == 1 ? W * 2 : W / 2, c4 = C >> 2;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * c4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(i % c4);
    const size_t pix = i / c4;
    const int xo = static_cast<int>(pix % Wo), yo = static_cast<int>((pix / Wo) % Ho);
    const int n = static_cast<int>(pix / (static_cast<size_t>(Wo) * Ho));
    float4 v;
    if (mode == 1) {
      v = ldg_f4(x + ((static_cast<size_t>(n) * H + (yo >> 1)) * W + (xo >> 1)) * C + cg * 4);
    } else {
      const float* b = x + ((static_cast<size_t>(n) * H + 2 * yo) * W + 2 * xo) * C + cg * 4;
      const float4 a0 = ldg_f4(b), a1 = ldg_f4(b + C), a2 = ldg_f4(b + static_cast<size_t>(W) * C), a3 = ldg_f4(b + static_cast<size_t>(W) * C + C);
      v = make_float4(((a0.x + a1.x) + (a2.x + a3.x)) * 0.25f, ((a0.y + a1.y) + (a2.y + a3.y)) * 0.25f,
                      ((a0.z + a1.z) + (a2.z + a3.z)) * 0.25f, ((a0.w + a1.w) + (a2.w + a3.w)) * 0.25f);
    }
    stg_f4(out + pix * C + cg * 4, v);
    if (out16 != nullptr) {
      uint2 pk;
      pk.x = pack_h2(v.x, v.y); pk.y = pack_h2(v.z, v.w);
      *reinterpret_cast<uint2*>(out16 + pix * C + cg * 4) = pk;
    }
  }
}

// Same-resolution GroupNorm apply over fp16 sources (ResBlock hidden tensor, fp16 copies of block outputs, virtual concat
// of two) with no raw outputs: the bulk of the element-wise traffic of a forward.  8 work items per trip kept packed
// (4 registers each) until consumed, so a thread has 128 bytes of reads in flight although an item is only 16 bytes.
// kHoist: the channel-group count divides the block size, so a thread keeps the same 8 channels on every trip and its 16
// coefficients live in registers (saves 16 shared-memory loads per 16-byte item).
// kF8: the activation is written as e4m3 to out_act8 (same element offsets).
template <bool kHoist, bool kLo = false, bool kF8 = false>
__global__ void __launch_bounds__(256, 3) gn_apply_h16_kernel(const GnApplyParams p) {
  extern __shared__ float s_ab[];
  __shared__ float s_mean[64], s_rstd[64];
  gn_prologue(p, s_ab, s_mean, s_rstd);
  const int C = p.C0 + p.C1, c8 = C >> 3, c80 = p.C0 >> 3;
  int n, bx;
  gn_block_pos(p, n, bx);
  const int HW = p.H * p.W;
  const int pix0 = bx * p.pix_per_block;
  const int npix = min(p.pix_per_block, HW - pix0);
  const int items = npix * c8;
  constexpr int U = 8;
  float A[8], B[8];
  if (kHoist) {
    const int cg = threadIdx.x % c8;
#pragma unroll
    for (int j = 0; j < 8; ++j) { A[j] = s_ab[j * c8 + cg]; B[j] = s_ab[C + j * c8 + cg]; }
  }
  auto apply8 = [&](const uint4& rawv, int cg, __half* dst) {
    const __half2* h2 = reinterpret_cast<const __half2*>(&rawv);
    uint32_t pk[4], pl[4];
    uint16_t p8[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h2[j]);
      float y0, y1;
      if (kHoist) {
        y0 = fmaf(f.x, A[2 * j], B[2 * j]);
        y1 = fmaf(f.y, A[2 * j + 1], B[2 * j + 1]);
      } else {
        y0 = fmaf(f.x, s_ab[(2 * j) * c8 + cg], s_ab[C + (2 * j) * c8 + cg]);
        y1 = fmaf(f.y, s_ab[(2 * j + 1) * c8 + cg], s_ab[C + (2 * j + 1) * c8 + cg]);
      }
      if (p.silu) { y0 = silu_f(y0); y1 = silu_f(y1); }
      if (kF8) { p8[j] = pack_e4m3x2(y0, y1); continue; }
      pk[j] = pack_h2(y0, y1);
      if (kLo) {
        const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&pk[j]));
        pl[j] = pack_h2(y0 - hi.x, y1 - hi.y);
      }
    }
    if (kF8) {
      *reinterpret_cast<uint2*>(p.out_act8 + (dst - p.out_act)) =
          make_uint2(p8[0] | (static_cast<uint32_t>(p8[1]) << 16), p8[2] | (static_cast<uint32_t>(p8[3]) << 16));
      return;
    }
    *reinterpret_cast<uint4*>(dst) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    if (kLo) *reinterpret_cast<uint4*>(p.out_lo + (dst - p.out_act)) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
  };
  if (kHoist) {
    // division-free addressing: the thread owns channel group cg and every (256 / c8)-th pixel starting at pr
    const int cg = threadIdx.x % c8, pr = threadIdx.x / c8, ppt = 256 / c8;
    const size_t px0 = static_cast<size_t>(n) * HW + pix0 + pr;
    const __half* src;
    size_t sstep;
    if (cg < c80) { src = p.x0h + px0 * p.C0 + cg * 8; sstep = static_cast<size_t>(ppt) * p.C0; }
    else { src = p.x1h + px0 * p.C1 + (cg - c80) * 8; sstep = static_cast<size_t>(ppt) * p.C1; }
    __half* dst = p.out_act + px0 * C + cg * 8;
    const size_t dstep = static_cast<size_t>(ppt) * C;
    int left = pr < npix ? (npix - pr + ppt - 1) / ppt : 0;      // pixels of this thread
    for (; left >= U; left -= U) {
      uint4 raw[U];
#pragma unroll
      for (int u = 0; u < U; ++u) raw[u] = __ldg(reinterpret_cast<const uint4*>(src + u * sstep));
#pragma unroll
      for (int u = 0; u < U; ++u) apply8(raw[u], cg, dst + u * dstep);
      src += U * sstep;
      dst += U * dstep;
    }
    for (; left > 0; --left) {
      apply8(__ldg(reinterpret_cast<const uint4*>(src)), cg, dst);
      src += sstep;
      dst += dstep;
    }
    return;
  }
  auto src_of = [&](int it) {
    const int cg = it % c8;
    const size_t px = static_cast<size_t>(n) * HW + pix0 + it / c8;
    return cg < c80 ? p.x0h + px * p.C0 + cg * 8 : p.x1h + px * p.C1 + (cg - c80) * 8;
  };
  auto finish = [&](int it, const uint4& rawv) {
    apply8(rawv, it % c8, p.out_act + (static_cast<size_t>(n) * HW + pix0 + it / c8) * C + (it % c8) * 8);
  };
  int it0 = threadIdx.x;
  for (; it0 + (U - 1) * 256 < items; it0 += U * 256) {
    uint4 raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) raw[u] = __ldg(reinterpret_cast<const uint4*>(src_of(it0 + u * 256)));
#pragma unroll
    for (int u = 0; u < U; ++u) finish(it0 + u * 256, raw[u]);
  }
  for (int it = it0; it < items; it += 256) finish(it, __ldg(reinterpret_cast<const uint4*>(src_of(it))));
}

// ----------------------------------------------------------------------------------------------
// network input: fp32 NCHW [Nx][Cin][H][W] -> fp16 NHWC [N][H][W][64]; sample n reads n % Nx (lets the two
// classifier-free-guidance halves share one x without a concat copy).
// The 64 operand channels carry a two-term split of the input, which the stem weights mirror (Unet::finalize):
//     channels [0,Cin) = hi = fp16(x)      [Cin,2Cin) = lo = fp16(x - hi)      [2Cin,3Cin) = hi      rest 0
//     weights            Wh                              Wh                                Wl
// so the stem computes  hi*Wh + lo*Wh + hi*Wl = x*W  to ~2^-21 at no extra cost (K is padded to 64 channels anyway):
// the input rounding of x_t would otherwise enter every layer coherently.
// One thread = 8 output channels (16 bytes) of one pixel.
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pack_input_kernel(const float* __restrict__ x, __half* __restrict__ out, int N,
                                                         int Nx, int Cin, int HW) {
  // phase 1: one thread per pixel reads its Cin fp32 values (coalesced along the pixel index of every channel plane);
  // phase 2: the block writes the 64 fp16 operand channels with 16-byte coalesced stores, one thread per (pixel, 8-channel group)
  __shared__ float s_ch[256][17];
  const size_t total = static_cast<size_t>(N) * HW;
  for (size_t base = blockIdx.x * static_cast<size_t>(blockDim.x); base < total; base += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t idx = base + threadIdx.x;
    if (idx < total) {
      const int n = static_cast<int>(idx / HW);
      const int p = static_cast<int>(idx % HW);
      const float* src = x + (static_cast<size_t>(n % Nx) * Cin) * HW + p;
#pragma unroll
      for (int c = 0; c < 16; ++c) s_ch[threadIdx.x][c] = c < Cin ? __ldg(src + static_cast<size_t>(c) * HW) : 0.f;
    }
    __syncthreads();
    const int live = static_cast<int>(min(static_cast<size_t>(256), total - base));
    for (int it = threadIdx.x; it < live * 8; it += 256) {
      const int px = it >> 3, g = it & 7;
      uint32_t w[4];
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
        w[k] = *reinterpret_cast<const uint32_t*>(&h2);
      }
      *reinterpret_cast<uint4*>(out + (base + px) * 64 + g * 8) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    __syncthreads();
  }
}

// ----------------------------------------------------------------------------------------------
// Output head, second half: eps[n][c][h][w] = bias[c] + sum over the 9 taps of Y[n][h+dy][w+dx][tap*Co + c].
// The 3x3 output convolution (adm.py:486, Cout = 4) is evaluated as a 1x1 GEMM with 9*Co output columns (one per tap and
// output channel: every activation element is read once instead of nine times) followed by this shift-and-add; taps that
// fall outside the image contribute nothing (zero padding).  Y is fp32 NHWC with row pitch ldy.
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) eps_gather_kernel(const float* __restrict__ Y, const float* __restrict__ bias,
                                                         float* __restrict__ eps, int N, int H, int W, int Co, int ldy) {
  const size_t total = static_cast<size_t>(N) * H * W;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int w = static_cast<int>(idx % W);
    const int h = static_cast<int>((idx / W) % H);
    const int n = static_cast<int>(idx / (static_cast<size_t>(W) * H));
    float acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;
    // summation order: tap 0..8 ascending (fixed, so results are bit-reproducible)
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int hh = h + tap / 3 - 1, ww = w + tap % 3 - 1;
      if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
      const float* src = Y + ((static_cast<size_t>(n) * H + hh) * W + ww) * ldy + tap * Co;
      if (Co == 4) {
        const float4 v = ldg_f4(src);
        acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w;
      } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) if (c < Co) acc[c] += __ldg(src + c);
      }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c)
      if (c < Co) eps[((static_cast<size_t>(n) * Co + c) * H + h) * W + w] = acc[c] + __ldg(bias + c);
  }
}

}  // namespace ivid
