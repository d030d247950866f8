// Fused QKV self-attention for head widths d = 64k, k >= 2 (attention_kernel in attention.cuh keeps d = 64).
//   reference: QKVAttention.forward adm.py:233-253 — per (sample, head): softmax_fp32((q*d^-1/4)^T (k*d^-1/4)) v,
//   legacy channel order [head][q|k|v][d] of the qkv projection (adm.py:246).
//
// Input : qkv  fp16 [N][T][3C]; head h owns channels [3dh, 3dh + 3d) = q|k|v.
// Output: o    fp16 [N][T][C]   channel = d*h + c.
//
// The same design as attention_kernel, generalised over d.  One CTA per (sample, head, 128-query tile, output-column slice),
// two warpgroups of 64 query rows each; thread 0 also streams 64-channel TMA boxes through an mbarrier ring in a fixed order.
// It refills a stage half a ring after that stage was released, so the two warpgroups may drift up to half a ring apart before
// the leading one waits for the other (attention_kernel refills at once, which keeps them in step).  256 threads leave up to
// 255 registers per thread for 4 x 32 O accumulators plus S and P (d = 128, NV = 2, fits 128 and runs two CTAs per SM).  Per key block of 64 keys a warpgroup
//   - builds S = Q K^T [64 x 64] in the same 32 accumulator registers as attention_kernel, contracting over d in k chunks of
//     64 channels (four m64n64k16 k-steps per chunk; ring step c holds K chunk c, plus Q chunk c when Q is streamed);
//   - turns S into fp16 probabilities P with the same lazy online softmax;
//   - accumulates O += P V for its slice of DV = 64 * nv output columns: nv ring steps, each one [64 keys x 64 ch] V box and
//     one m64n64k16 group of 32 accumulator registers (NV groups in registers, nv <= NV used by this slice).
// Slices: k <= 4 chunks (d <= 256) is one slice.  Above that the output columns are split into ceil(k/4) slices of at most
// NV <= 4 boxes each (the last one may be narrower), and every slice's CTA recomputes S over the full d.  The QK^T work is
// therefore done ceil(k/4) times instead of once — 2x at d = 512, 4x at d = 1024 — which raises the attention FLOPs by
// (ceil(k/4) + 1) / 2 (1.5x at d = 512, 2.5x at d = 1024); attention is ~2 % of a forward (DESIGN.md §4).
// Q staging: for k <= 8 (d <= 512, <= 128 KB) Q stays resident in shared memory, loaded once; above that each S ring step
// also carries the 128 x 64 Q chunk next to its K chunk (Q is re-read from L2 once per key block).
// Scale: (q*s)(k*s) with s = d^-1/4 is evaluated as (q.k) * (d^-1/2 * log2 e) in fp32.  For d = 64, s^2 = 0.125 is an exact
// power of two and both forms scale exactly; for other widths s is not a power of two (d^-1/2 is not even one for d = 128,
// 192, 512), so the logits differ from the reference's form by a few fp32 roundings — far below the fp16 operand rounding.
// No atomics and a fixed reduction order: the result is bitwise reproducible and independent of the batch.
#pragma once
#include "attention.cuh"
#include "common.cuh"

namespace ivid {

struct AttnHdParams {
  int N, T, C, d, heads;
  int chunks;          // d / 64
  int q_tiles;         // ceil(T / 128)
  int slices;          // output-column slices of NV boxes (the last may hold fewer)
  int stages;          // ring depth
  float scale_log2;    // d^-1/2 * log2(e)
  __half* out;         // [N][T][C]
};

struct AttnHdCfg {
  static constexpr int KV = 64;
  static constexpr int BOX_BYTES = 64 * 64 * 2;                  // one [64 rows x 64 ch] fp16 box
  static constexpr int QCHUNK_BYTES = 128 * 64 * 2;              // [128 query rows x 64 ch]
  static constexpr int THREADS = 256;
  static constexpr int MAX_STAGES = 16;
  static constexpr int MAX_SMEM = 227 * 1024;
  static constexpr int MAX_SMEM_2CTA = 113 * 1024;               // NV = 2 (d = 128): two CTAs per SM, <= 128 registers
  static constexpr int RESIDENT_Q_MAX_CHUNKS = 8;                // Q resident up to d = 512 (128 KB)
  static constexpr int stage_bytes(bool qres) { return qres ? BOX_BYTES : BOX_BYTES + QCHUNK_BYTES; }
};

template <int NV, bool QRES>
__global__ void __launch_bounds__(AttnHdCfg::THREADS, NV == 2 ? 2 : 1)
attention_hd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapKV, const AttnHdParams p) {
  using Cfg = AttnHdCfg;
  constexpr int STAGE = Cfg::stage_bytes(QRES);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;                                               // QRES: chunk c at c * QCHUNK_BYTES
  uint8_t* sStg = smem + (QRES ? p.chunks * Cfg::QCHUNK_BYTES : 0);  // stage s at s * STAGE: K or V box, then (!QRES) Q chunk
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStg + p.stages * STAGE);
  uint64_t* q_full = bars;
  uint64_t* full = bars + 1;                // [stages]
  uint64_t* empty = full + Cfg::MAX_STAGES; // [stages]

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;
  int b = blockIdx.x;
  const int qt = b % p.q_tiles; b /= p.q_tiles;
  const int slice = b % p.slices; b /= p.slices;
  const int head = b % p.heads;
  const int n = b / p.heads;
  const int nkv = (p.T + Cfg::KV - 1) / Cfg::KV;
  const int kv_tail = p.T - (nkv - 1) * Cfg::KV;                    // valid keys of the last block (see mask_key_tail)
  const int nv = min(NV, p.chunks - slice * NV);                    // V boxes of this slice (>= 1)
  const int q_ch = head * 3 * p.d, k_ch = q_ch + p.d, v_ch = q_ch + 2 * p.d + slice * NV * 64;

  // ring step i of key block j = i / P (P = k + nv steps per block): K chunk i % P (with its Q chunk when Q is streamed) for
  // i % P < k, else V box i % P - k.  Step i uses stage i % NS.
  const int NS = p.stages, P = p.chunks + nv, total = nkv * P, lag = NS / 2;
  auto load_step = [&](int i) {
    const int st = i % NS, round = i / NS, j = i / P, r = i - j * P;
    if (round > 0) mbar_wait(&empty[st], (round - 1) & 1);
    uint8_t* dst = sStg + st * STAGE;
    if (r < p.chunks) {
      mbar_arrive_expect_tx(&full[st], STAGE);
      tma_load_3d(&mapKV, &full[st], dst, k_ch + 64 * r, j * Cfg::KV, n);
      if (!QRES) tma_load_3d(&mapQ, &full[st], dst + Cfg::BOX_BYTES, q_ch + 64 * r, qt * 128, n);
    } else {
      mbar_arrive_expect_tx(&full[st], Cfg::BOX_BYTES);
      tma_load_3d(&mapKV, &full[st], dst, v_ch + 64 * (r - p.chunks), j * Cfg::KV, n);
    }
  };
  if (tid == 0) {
    tma_prefetch_desc(&mapQ);
    tma_prefetch_desc(&mapKV);
    mbar_init(q_full, 1);
    for (int s = 0; s < NS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }   // empty: one arrive per warp
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    if (QRES) {
      mbar_arrive_expect_tx(q_full, p.chunks * Cfg::QCHUNK_BYTES);
      for (int c = 0; c < p.chunks; ++c) tma_load_3d(&mapQ, q_full, sQ + c * Cfg::QCHUNK_BYTES, q_ch + 64 * c, qt * 128, n);
    }
    for (int i = 0; i < NS && i < total; ++i) load_step(i);
  }

  // warpgroup wg owns query rows [qt*128 + 64wg, +64).  Steps are waited for (st, ph) and released (rel) in order.
  int st = 0, rel = 0;
  uint32_t ph = 0;
  auto advance = [&]() { if (++st == NS) { st = 0; ph ^= 1u; } };
  auto release = [&]() {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[rel % NS]);
    if (tid == 0 && rel >= lag && rel + NS - lag < total) load_step(rel + NS - lag);
    __syncwarp();
    ++rel;
  };
  const float kScaleLog2 = p.scale_log2;
  constexpr float kLazy = 8.0f;        // see attention_kernel
  float o[NV][32];
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[v][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};     // rows lane/4 and lane/4 + 8 of the warp
  if (QRES) mbar_wait(q_full, 0);
#pragma unroll 1
  for (int j = 0; j < nkv; ++j) {
    // S = Q K^T over k chunks; the stage of chunk c - 1 is released once chunk c is issued and c - 1 has completed
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.f;
#pragma unroll 1
    for (int c = 0; c < p.chunks; ++c) {
      mbar_wait(&full[st], ph);
      const uint32_t stage = smem_u32(sStg + st * STAGE);
      const uint32_t q_addr = QRES ? smem_u32(sQ + c * Cfg::QCHUNK_BYTES) : stage + Cfg::BOX_BYTES;
      const uint64_t dq = make_smem_desc_sw128(q_addr + wg * 64 * 128, 1024, 16);
      const uint64_t dk = make_smem_desc_sw128(stage, 1024, 16);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_ss<64>(s, dq + 2 * k, dk + 2 * k, 1u);
      wgmma_commit();
      if (c > 0) {
        wgmma_wait<1>();
        release();
      }
      advance();
    }
    wgmma_wait<0>();
    reg_fence(s);
    release();
    if (j == nkv - 1 && kv_tail != Cfg::KV) mask_key_tail(s, kv_tail, lane);
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
      m_new[r] = (m_cand - m_run[r] > kLazy) ? m_cand : m_run[r];
      alpha[r] = ex2_ftz(m_run[r] - m_new[r]);
      m_run[r] = m_new[r];
    }
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
      for (int v = 0; v < NV; ++v)
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          o[v][4 * c] *= alpha[0]; o[v][4 * c + 1] *= alpha[0];
          o[v][4 * c + 2] *= alpha[1]; o[v][4 * c + 3] *= alpha[1];
        }
    }
    // O += P V, one 64-column group per V box
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      if (v < nv) {
        mbar_wait(&full[st], ph);
        const uint64_t dv = make_smem_desc_sw128(smem_u32(sStg + st * STAGE), 1024, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_rs_tb<64>(o[v], pa[k], dv + 128 * k, 1u);
        wgmma_commit();
        if (v > 0) {
          wgmma_wait<1>();
          release();
        }
        advance();
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int v = 0; v < NV; ++v) reg_fence(o[v]);
    release();
  }
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
    __half* out = p.out + (static_cast<size_t>(n) * p.T + t) * p.C + head * p.d + slice * NV * 64 + 2 * (lane & 3);
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      if (v < nv) {
#pragma unroll
        for (int c = 0; c < 8; ++c)
          *reinterpret_cast<uint32_t*>(out + 64 * v + 8 * c) = pack_h2(o[v][4 * c + 2 * r] * inv, o[v][4 * c + 2 * r + 1] * inv);
      }
    }
  }
}

}  // namespace ivid
