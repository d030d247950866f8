// Fused QKV self-attention core (FlashAttention-style, no T x T matrix in HBM) on Hopper wgmma.
//   reference: QKVAttention.forward adm.py:233-253 — per (sample, head): softmax_fp32((q*d^-1/4)^T (k*d^-1/4)) v,
//   legacy channel order [head][q|k|v][64] of the qkv projection (adm.py:246), head dim 64.
//
// Input : qkv  fp16 [N][T][3C]  (NHWC output of the qkv 1x1 GEMM); head h owns channels [192h, 192h+192) = q|k|v.
// Output: o    fp16 [N][T][C]   channel = 64*h + d   (== reshape(bs, -1, length) of the reference).
//
// One CTA per (sample, head, 128-query tile), two warpgroups of 64 query rows each, 64 keys per step.  Thread 0 drives a
// four-deep TMA ring of K / V tiles shared by both warpgroups.  Per key block a warpgroup computes S = Q K^T into
// registers (wgmma, Q and K from shared memory), turns it into un-normalised fp16 probabilities P in place and
// accumulates O += P V with P as the register A operand (its fragment layout is the accumulator's) and V as an MN-major
// shared-memory operand; the online-softmax rescale of O happens in registers.  (q*s)(k*s) with s = 64^-1/4 is
// evaluated as (q.k) * 0.125 — an exact power of two.
// Any T >= 1: ceil(T / 64) key blocks; TMA zero-fills K / V / Q rows past T (the tensor map's T dimension keeps them inside
// the sample), the last block's keys >= T are masked to -inf (mask_key_tail) and query rows >= T are not stored.
#pragma once
#include "common.cuh"

namespace ivid {

struct AttnParams {
  int N, T, C, heads;
  int q_tiles;        // ceil(T / 128)
  __half* out;        // [N][T][C]
};

struct AttnCfg {
  static constexpr int KV = 64;
  static constexpr int Q_BYTES = 128 * 64 * 2;
  static constexpr int KV_BYTES = KV * 64 * 2;
  static constexpr int STAGES = 4;
  static constexpr int SMEM_BYTES = Q_BYTES + STAGES * 2 * KV_BYTES + 1024 /*barriers*/ + 1024 /*align*/;
  static constexpr int THREADS = 256;
};

// 2^x on the SFU without exp2f()'s denormal pre/post-scaling: inputs here are <= 0 after the running-maximum subtraction,
// results below 2^-126 flush to 0 and contribute nothing to a sum whose largest term is >= 2^-8.
__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Sequence tail (T % 64 != 0): the last key block's rows >= T are TMA zero fill; their logits are set to -inf before the row
// maximum, so their probabilities are exactly 0.  Accumulator group c of a thread holds key columns 8c + 2(lane & 3) + {0, 1}
// for both of its rows.  Applied on that block only, so sequences of whole blocks keep their bits.
__device__ __forceinline__ void mask_key_tail(float (&s)[32], int valid, int lane) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int col = 8 * c + 2 * (lane & 3);
    if (col >= valid) { s[4 * c] = -INFINITY; s[4 * c + 2] = -INFINITY; }
    if (col + 1 >= valid) { s[4 * c + 1] = -INFINITY; s[4 * c + 3] = -INFINITY; }
  }
}

__global__ void __launch_bounds__(256, 2)
attention_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapKV, const AttnParams p) {
  using Cfg = AttnCfg;
  constexpr int KV = Cfg::KV, ST = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sKV = smem + Cfg::Q_BYTES;                       // stage s: K at sKV + s*2*KV_BYTES, V right after
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + ST * 2 * Cfg::KV_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;          // [ST]
  uint64_t* kv_empty = kv_full + ST;     // [ST]

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  const int qt = blockIdx.x % p.q_tiles;
  const int head = (blockIdx.x / p.q_tiles) % p.heads;
  const int n = blockIdx.x / (p.q_tiles * p.heads);
  const int nkv = (p.T + KV - 1) / KV;
  const int kv_tail = p.T - (nkv - 1) * KV;                 // valid keys of the last block (KV unless T % 64 != 0)

  auto load_kv = [&](int j) {
    const int st = j % ST;
    if (j >= ST) mbar_wait(&kv_empty[st], ((j / ST) - 1) & 1);
    uint8_t* sk = sKV + st * 2 * Cfg::KV_BYTES;
    mbar_arrive_expect_tx(&kv_full[st], 2 * Cfg::KV_BYTES);
    tma_load_3d(&mapKV, &kv_full[st], sk, head * 192 + 64, j * KV, n);
    tma_load_3d(&mapKV, &kv_full[st], sk + Cfg::KV_BYTES, head * 192 + 128, j * KV, n);
  };
  if (tid == 0) {
    tma_prefetch_desc(&mapQ);
    tma_prefetch_desc(&mapKV);
    mbar_init(q_full, 1);
    for (int s = 0; s < ST; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 8); }      // kv_empty: one arrive per warp
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(q_full, Cfg::Q_BYTES);
    tma_load_3d(&mapQ, q_full, sQ, head * 192, qt * 128, n);
    for (int j = 0; j < ST && j < nkv; ++j) load_kv(j);
  }

  constexpr float kScaleLog2 = 0.125f * 1.4426950408889634f;   // (64^-1/4)^2 * log2(e)
  // lazy online softmax: the reference maximum of a row only moves when the new maximum exceeds it by more than 2^kLazy
  // (probabilities stay <= 2^kLazy, far inside fp16 range, and O / l does not depend on the reference)
  constexpr float kLazy = 8.0f;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};     // rows lane/4 and lane/4 + 8 of the warp
  mbar_wait(q_full, 0);
  const uint64_t dq = make_smem_desc_sw128(smem_u32(sQ) + wg * 64 * 128, 1024, 16);
#pragma unroll 1
  for (int j = 0; j < nkv; ++j) {
    const int st = j % ST;
    mbar_wait(&kv_full[st], (j / ST) & 1);
    const uint32_t sk = smem_u32(sKV + st * 2 * Cfg::KV_BYTES);
    const uint64_t dk = make_smem_desc_sw128(sk, 1024, 16);
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss<64>(s, dq + 2 * k, dk + 2 * k, k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    if (j == nkv - 1 && kv_tail != KV) mask_key_tail(s, kv_tail, lane);
    // row maxima: a thread holds 16 columns of each of its two rows; the four lanes of a row combine theirs
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      mx[0] = fmaxf(mx[0], fmaxf(s[4 * c], s[4 * c + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[4 * c + 2], s[4 * c + 3]));
    }
    float alpha[2], m_new[2], lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_cand = fmaxf(m_run[r], mx[r] * kScaleLog2);
      m_new[r] = (m_cand - m_run[r] > kLazy) ? m_cand : m_run[r];      // m_run = -inf on the first block: always taken
      alpha[r] = ex2_ftz(m_run[r] - m_new[r]);
      m_run[r] = m_new[r];
    }
    // P (fp16) as the A operand of P V: K step k covers key columns [16k, 16k + 16) = accumulator groups 2k and 2k + 1
    uint32_t pa[4][4];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float p0 = ex2_ftz(s[4 * c] * kScaleLog2 - m_new[0]), p1 = ex2_ftz(s[4 * c + 1] * kScaleLog2 - m_new[0]);
      const float p2 = ex2_ftz(s[4 * c + 2] * kScaleLog2 - m_new[1]), p3 = ex2_ftz(s[4 * c + 3] * kScaleLog2 - m_new[1]);
      lsum[0] += p0 + p1;
      lsum[1] += p2 + p3;
      pa[c >> 1][(c & 1) * 2 + 0] = pack_h2(p0, p1);
      pa[c >> 1][(c & 1) * 2 + 1] = pack_h2(p2, p3);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + lsum[r];
    if (alpha[0] != 1.0f || alpha[1] != 1.0f) {
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        o[4 * c] *= alpha[0]; o[4 * c + 1] *= alpha[0];
        o[4 * c + 2] *= alpha[1]; o[4 * c + 3] *= alpha[1];
      }
    }
    // V tile [KV rows][64 d] is an MN-major B operand: 16 kv rows (one MMA K step) = 2048 B
    const uint64_t dv = make_smem_desc_sw128(sk + Cfg::KV_BYTES, 1024, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_rs_tb<64>(o, pa[k], dv + 128 * k, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
    if (tid == 0 && j + ST < nkv) load_kv(j + ST);
  }
  // row sums: combine the four lanes of each row
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int t = qt * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
    if (t >= p.T) continue;
    const float inv = 1.0f / l_run[r];
    __half* out = p.out + (static_cast<size_t>(n) * p.T + t) * p.C + head * 64 + 2 * (lane & 3);
#pragma unroll
    for (int c = 0; c < 8; ++c)
      *reinterpret_cast<uint32_t*>(out + 8 * c) = pack_h2(o[4 * c + 2 * r] * inv, o[4 * c + 2 * r + 1] * inv);
  }
}

// Perturbed-attention rows (PAG, Ahn et al. 2024, arXiv:2403.17377): the attention map is replaced by the identity, so the
// output of each head is its V channels, copied bit for bit.  Rows [row0, N) of qkv [N][T][3C] (head h of width d owns q|k|v
// at channels [3dh, 3dh + 3d)) -> out [N][T][C] channel dh + c = qkv channel 3dh + 2d + c.  One 16-byte group of 8 channels
// per work item (C and d are multiples of 64, so a group never straddles a head).
__global__ void __launch_bounds__(256) attention_identity_kernel(const __half* __restrict__ qkv, __half* __restrict__ out,
                                                                 size_t row0, size_t rows, int C, int d) {
  const int groups = C / 8;
  const size_t items = rows * groups;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < items; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t row = row0 + i / groups;                  // n * T + t
    const int c8 = static_cast<int>(i % groups) * 8;
    const int h = c8 / d, c = c8 - h * d;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(qkv + row * 3 * C + 3 * d * h + 2 * d + c));
    *reinterpret_cast<uint4*>(out + row * C + c8) = v;
  }
}

}  // namespace ivid
