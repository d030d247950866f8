// Implicit-GEMM convolution (3x3 pad 1 / 1x1) for NHWC fp16 activations on Hopper wgmma tensor cores.
//
// Replaces, on the ADM UNet hot path, every nn.Conv2d / nn.Conv1d the reference issues through cuDNN:
//   ResBlock2d in_layers[2] / out_layers[3] / skip_connection   (reference diffusion/backbones/adm.py:160,182,190)
//   AttentionBlock qkv / proj_out                                (adm.py:275,278)
//   input conv / final out conv                                  (adm.py:369,486)
//
// GEMM view:  D[M = N*H*W pixels, Cout] = A[M, K] * B[Cout, K]^T,   K = sum over segments of taps*C_seg.
//   A is never materialised (no im2col buffer): for every filter tap one 4-D TMA box load (64 channels x TW x TH x TN
//   pixels) at the tap-shifted coordinate; TMA's out-of-bounds zero fill implements the conv zero padding.  Further
//   "segments" let a 1x1 skip convolution over a different tensor (raw x) accumulate into the same tile as extra K slabs
//   (SURVEY K2), so  skip(x) + conv(h)  is one kernel.
//   B (weights) is packed [Cout_pad][K] fp16, K-major, by conv_pack (ops.cu) on the host, and loaded by 2-D TMA.
//   Segments of C % 64 != 0 channels (C % 8 == 0) run ceil(C/64) chunks: the activation map keeps the real channel extent, so
//   TMA zero-fills the channels past C of the last box, and the packed weights hold zero columns there.  Out-of-bounds
//   elements still count toward the transaction bytes, so every stage expects the full box.
// Both operands land in shared memory in the 128-byte-swizzled K-major layout that wgmma reads directly.
//
// Every CTA computes one 128-pixel x BN output tile.  Block b takes pixel tile b / n_blocks and column block b % n_blocks, so
// the CTAs that share an activation tile run together.  Two consumer warpgroups per CTA (rows 0-63 / 64-127 of the tile),
// accumulators in registers, and one producer warp (warp 8) whose elected lane drives the TMA ring: it runs STAGES k-blocks
// ahead and refills a slot as soon as all eight consumer warps have released it.  A consumer keeps one wgmma group in
// flight: it issues the group of k-block u, waits for group u - 1 to retire and only then releases u - 1's slot, so its
// tensor work never stops for a refill.  Two CTAs fit one SM (BN <= 128), so one CTA's epilogue overlaps the other's main
// loop.
// The epilogue adds bias and residual (optionally through a nearest-2x upsample) to the accumulator fragments and writes
// fp32 / fp16 / NCHW output, an optional fp16 copy and the per-(sample, channel) GroupNorm statistics of the output.  The
// ring is idle by then, so it holds the staged NHWC tile (ConvGemmCfg): the residual's boxes arrive in it by TMA as extra
// k-blocks behind the last operand loads, and the outputs leave it by TMA box stores, issued by one thread.
//
// Slab mode (SLAB, chosen by conv_launch_create for tiles of one sample and TW >= 8): the three taps of a 3x3 segment that
// differ only in dy read the same pixels shifted by one image row.  So the producer loads one (TH + 2)-row activation slab
// per (chunk, dx), box (64 ch, TW, TH + 2, 1) at row h0 - 1, and the k-blocks of dy = -1, 0, 1 start their A descriptor 0,
// TW*128 and 2*TW*128 bytes into it.  TW*128 is a whole number of 1024-byte swizzle atoms when TW >= 8, so a shifted start
// sees exactly the layout of a box loaded at that row.  K runs chunk slow, then dx, then dy fastest; the packed weight
// columns are the same as per tap.  The slabs have a ring of their own (2 slots, released after the third dy's group has
// retired); the weight boxes keep a per-k-block ring, 4 deep.  A 1x1 segment of a slab launch puts its one box per chunk in
// a slab slot.  Per three k-blocks a CTA takes in TW*(TH+2)*128 + 3*BN*128 bytes instead of 3*(16 KB + BN*128).  The
// epilogue's staging and statistics scratch lie over the ring, which is idle once both warpgroups' last groups have retired.
//
// fp8 operand mode (A8): segment 0 is e4m3.  Its 128-byte box row is 128 channels, so an e4m3 k-block has exactly the
// shared-memory layout, TMA bytes and wgmma descriptors of an fp16 one; only the instruction differs (k32 e4m3 for k16
// f16) and a chunk covers 128 channels.  Its weights come from a second map (b8) over e4m3 columns pre-scaled by 2^e; the
// fp16 skip segments keep the b map with columns pre-scaled by the same 2^e, so all of K sums into one accumulator, and
// the epilogue takes v = acc * 2^-e + bias.  conv_pack writes both and decides which convs qualify.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace ivid {

struct ConvGemmParams {
  int N, H, W;                 // batch and spatial size of the conv input == output (stride 1)
  int TW, TH, TN;              // pixel tile (TW*TH*TN == 128)
  int tiles_w, tiles_h, tiles_n;
  int n_blocks;                // Cout_pad / BN
  int seg_chunks[3];           // ceil(channels/64) of each K segment (0 = segment unused)
  int seg_taps[3];             // 9 (3x3) or 1 (1x1)
  int Cout;                    // valid output channels
  int ldc;                     // output channel stride (elements) for NHWC modes
  int ldr;                     // residual channel stride (elements)
  int out_mode;                // 0 = fp32 NHWC, 1 = fp16 NHWC, 2 = fp32 NCHW (Cout planes)
  const float* bias;           // [Cout_pad] fp32
  const float* residual;       // fp32 NHWC or nullptr
  int res_up;                  // the residual is the nearest-2x upsample of a [N][H/2][W/2][ldr] tensor
  void* out;
  __half* out16;               // optional fp16 NHWC copy of an fp32 NHWC output (same ldc)
  double* stats;               // optional [N][Cout][2] per-(sample, channel) sum / sum-of-squares of the output (GroupNorm);
                               // of the ROUNDED values when the output is fp16 (exactly what the next GroupNorm reads)
  float acc_scale;             // A8 only: 2^-e, the inverse of the weights' power-of-two scale
};

// All TMA descriptors of one launch, passed as a single __grid_constant__ argument.
struct ConvMaps {
  CUtensorMap a[3];            // activation segments (fp16 NHWC)
  CUtensorMap b;               // packed weights
  CUtensorMap r;               // fp32 residual, box (F32_CH, TW, TH, TN); under res_up the half-size source tile
  CUtensorMap o;               // fp32 NHWC output, box (F32_CH, TW, TH, TN)
  CUtensorMap o16;             // fp16 NHWC output or copy, box (F16_CH, TW, TH, TN)
};
// the A8 kernels' maps: also the e4m3 weight columns of segment 0
struct ConvMaps8 : ConvMaps {
  CUtensorMap b8;
};

template <int BN, bool SLAB = false>
struct ConvGemmCfg {
  static constexpr int BM = 128;
  static constexpr int BK = 64;
  static constexpr int A_BYTES = BM * BK * 2;                  // 16 KB
  static constexpr int B_BYTES = ((BN * BK * 2 + 1023) / 1024) * 1024;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = BN == 128 && !SLAB ? 3 : 4;   // k-blocks in flight (SLAB: weight boxes)
  // SLAB: the largest slab, TW * (TH + 2) pixels with TW * TH = 128 and TW >= 8 (16 x 10), in each of 2 slots.  Two CTAs
  // of 2 slabs + 4 weight boxes (BN 128: 104 KB) fit one SM only with the statistics scratch over the ring; a third slab
  // or a third weight box in its place measured slower.
  static constexpr int SLAB_BYTES = 16 * 10 * 128;
  static constexpr int SLAB_STAGES = 2;
  static constexpr int RING_BYTES = SLAB ? SLAB_STAGES * SLAB_BYTES + STAGES * B_BYTES : STAGES * STAGE_BYTES;
  static constexpr int BAR_BYTES = 128;
  static constexpr int STAT_BYTES = 8 * 2 * BN * 4;            // [8 warps][sum|sumsq][BN] fp32
  static constexpr bool STATS_ON_RING = SLAB;                  // the epilogue's statistics scratch over the idle ring
  static constexpr int SMEM_BYTES = RING_BYTES + BAR_BYTES + (STATS_ON_RING ? 0 : STAT_BYTES) + 1024;   // +1024 alignment slack
  static constexpr int CONSUMER_THREADS = 256;                 // two warpgroups: MMA and epilogue
  static constexpr int THREADS = CONSUMER_THREADS + 32;        // + one producer warp: TMA loads

  // Epilogue staging over the idle ring.  The fp32 tile is UNITS units of UNIT_BOXES boxes (F32_CH channels x 128 pixels,
  // one F32_CH * 4-byte row per pixel, swizzled over that row); the residual's units arrive as k-blocks nunits, nunits + 1,
  // ... in the slots those take.  SLAB: a unit is a weight slot (F32_CH = BN / 4) and there are STAGES of them, so unit q
  // is the one k-block nunits + i with (nunits + i) % STAGES == q brings into slot q; the fp16 tile and the statistics
  // lie over the slab slots.  Per tap: unit u is the front of stage (nunits + u) % STAGES, and the fp16 tile fills stage
  // (nunits + UNITS) % STAGES.
  static constexpr int F32_CH = SLAB ? BN / 4 : (BN < 32 ? BN : 32);
  static constexpr int F32_BOX = BM * F32_CH * 4;
  static constexpr int UNIT_BOXES = !SLAB && BN == 128 ? 2 : 1;
  static constexpr int UNIT_CH = F32_CH * UNIT_BOXES;
  static constexpr int UNITS = BN / UNIT_CH;
  static constexpr int UNIT_STRIDE = SLAB ? B_BYTES : STAGE_BYTES;
  static constexpr int F16_CH = BN < 64 ? BN : 64;             // fp16 tile: BN / F16_CH boxes of F16_CH channels
  static constexpr int F16_BOX = BM * F16_CH * 2;
  static constexpr int F16_TILE = BM * BN * 2;
  static_assert(UNIT_BOXES * F32_BOX <= UNIT_STRIDE, "an fp32 unit must fit its ring slot");
  static_assert(SLAB ? UNITS == STAGES : UNITS < STAGES && F16_TILE <= STAGE_BYTES, "fp32 units and the fp16 tile must fit the ring");
  static_assert(!SLAB || F16_TILE + STAT_BYTES <= SLAB_STAGES * SLAB_BYTES, "the fp16 tile and statistics must fit the slab slots");
};

// position in the K loop: segment, tap, 64-channel chunk, and the first packed weight column of the segment
struct ConvKCursor {
  int seg = 0, t = 0, ch = 0, base = 0;
};

// p is read in place (__grid_constant__): the K cursor indexes seg_chunks / seg_taps at run time, and without it the compiler
// may copy the whole struct to a local-memory stack frame to do so.
template <int BN, bool A8 = false, bool SLAB = false>
__global__ void __launch_bounds__(ConvGemmCfg<BN>::THREADS, 2)
conv_gemm_kernel(const __grid_constant__ std::conditional_t<A8, ConvMaps8, ConvMaps> maps, const __grid_constant__ ConvGemmParams p) {
  using Cfg = ConvGemmCfg<BN, SLAB>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int SLAB_STAGES = Cfg::SLAB_STAGES;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (128-byte swizzle atoms) by pointer arithmetic on the __shared__ array
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::RING_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* slab_full = empty_bar + STAGES;      // SLAB only
  uint64_t* slab_empty = slab_full + SLAB_STAGES;
  float* stat_smem = reinterpret_cast<float*>(Cfg::STATS_ON_RING ? smem + Cfg::F16_TILE : smem + Cfg::RING_BYTES + Cfg::BAR_BYTES);
  uint8_t* const slab_ring = smem;               // SLAB: [SLAB_STAGES][SLAB_BYTES], then [STAGES][B_BYTES] weight boxes
  uint8_t* const w_ring = smem + SLAB_STAGES * Cfg::SLAB_BYTES;

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;                      // consumer warpgroup: tile rows [64 wg, 64 wg + 64)

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8u);              // one arrive per consumer warp
    }
    if constexpr (SLAB) {
      for (int s = 0; s < SLAB_STAGES; ++s) {
        mbar_init(&slab_full[s], 1);
        mbar_init(&slab_empty[s], 8u);
      }
    }
    fence_barrier_init();
  }
  __syncthreads();

  int nunits = 0;                                // K blocks of the tile
  for (int sg = 0; sg < 3; ++sg) nunits += p.seg_chunks[sg] * p.seg_taps[sg];
  const int nunits8 = A8 ? p.seg_chunks[0] * p.seg_taps[0] : 0;   // the first nunits8 k-blocks are e4m3

  // column block fast: the CTAs that share an activation tile run together
  const int mt = static_cast<int>(blockIdx.x) / p.n_blocks, nb = static_cast<int>(blockIdx.x) % p.n_blocks;
  const int colbase = nb * BN;
  const int tiles_per_img = p.tiles_w * p.tiles_h;
  const int tn = mt / tiles_per_img;
  const int rem = mt - tn * tiles_per_img;
  const int th = rem / p.tiles_w;
  const int tw = rem - th * p.tiles_w;
  const int n0 = tn * p.TN, h0 = th * p.TH, w0 = tw * p.TW;
  uint8_t* const unit_ring = SLAB ? w_ring : smem;                  // the epilogue's fp32 units

  // ===================================== producer warp =====================================
  if (warp == Cfg::CONSUMER_THREADS / 32) {
    if (lane == 0) {
      // residual box origin: under res_up the nearest-2x source tile at half the coordinates
      const int rw0 = p.res_up ? w0 >> 1 : w0, rh0 = p.res_up ? h0 >> 1 : h0;
      tma_prefetch_desc(&maps.a[0]);
      tma_prefetch_desc(&maps.b);
      if constexpr (A8) tma_prefetch_desc(&maps.b8);
      // the residual is read only after the main loop: start it towards L2 now
      if (p.residual != nullptr) {
#pragma unroll
        for (int q = 0; q < Cfg::UNITS * Cfg::UNIT_BOXES; ++q) tma_prefetch_l2_4d(&maps.r, colbase + q * Cfg::F32_CH, rw0, rh0, n0);
      }
      if constexpr (SLAB) {
        // per segment: chunk slow, dx, dy fast (3x3: one slab per (chunk, dx)); 1x1: one box per chunk
        const uint32_t slab_bytes = static_cast<uint32_t>(p.TW * (p.TH + 2)) * 128u;
        uint32_t u = 0, a = 0;                     // k-block, activation load
        int base = 0;
#pragma unroll 1
        for (int sg = 0; sg < 3; ++sg) {
          const int chunks = p.seg_chunks[sg];
          const int nx = p.seg_taps[sg] == 9 ? 3 : 1;
          const bool e4m3 = A8 && sg == 0;         // 128 channels per box row; columns of b8 (base stays 0)
#pragma unroll 1
          for (int ch = 0; ch < chunks; ++ch) {
#pragma unroll 1
            for (int xi = 0; xi < nx; ++xi, ++a) {
              const int sl = static_cast<int>(a % SLAB_STAGES);
              if (a >= SLAB_STAGES) mbar_wait(&slab_empty[sl], ((a / SLAB_STAGES) - 1) & 1);
              mbar_arrive_expect_tx(&slab_full[sl], nx == 3 ? slab_bytes : static_cast<uint32_t>(Cfg::A_BYTES));
              tma_load_4d(&maps.a[sg], &slab_full[sl], slab_ring + sl * Cfg::SLAB_BYTES, ch * (e4m3 ? 128 : 64),
                          w0 + (nx == 3 ? xi - 1 : 0), h0 - (nx == 3 ? 1 : 0), n0);
#pragma unroll 1
              for (int yi = 0; yi < nx; ++yi, ++u) {
                const int s = static_cast<int>(u % STAGES);
                if (u >= STAGES) mbar_wait(&empty_bar[s], ((u / STAGES) - 1) & 1);
                mbar_arrive_expect_tx(&full_bar[s], BN * Cfg::BK * 2);
                const int t = nx == 3 ? 3 * yi + xi : 0;
                uint8_t* sb = w_ring + s * Cfg::B_BYTES;
                if constexpr (A8) {
                  if (e4m3) { tma_load_2d(&maps.b8, &full_bar[s], sb, (t * chunks + ch) * 128, colbase); continue; }
                }
                tma_load_2d(&maps.b, &full_bar[s], sb, base + (t * chunks + ch) * 64, colbase);
              }
            }
          }
          if (!e4m3) base += p.seg_taps[sg] * chunks * 64;
        }
      } else {
        ConvKCursor c;                            // units are issued strictly in order: segment, tap slow, chunk fast
        while (p.seg_chunks[c.seg] == 0) ++c.seg;
#pragma unroll 1
        for (int u = 0; u < nunits; ++u) {
          const uint32_t g = static_cast<uint32_t>(u);
          const int s = static_cast<int>(g % STAGES);
          if (g >= STAGES) mbar_wait(&empty_bar[s], ((g / STAGES) - 1) & 1);
          const int taps = p.seg_taps[c.seg], chunks = p.seg_chunks[c.seg];
          uint8_t* sa = smem + s * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + Cfg::A_BYTES;
          const int dy = (taps == 9) ? (c.t / 3 - 1) : 0;
          const int dx = (taps == 9) ? (c.t % 3 - 1) : 0;
          mbar_arrive_expect_tx(&full_bar[s], Cfg::A_BYTES + BN * Cfg::BK * 2);
          bool e4m3 = false;
          if constexpr (A8) {
            if (c.seg == 0) {                      // e4m3: 128 channels per box row; columns of b8 (c.base stays 0)
              tma_load_4d(&maps.a[0], &full_bar[s], sa, c.ch * 128, w0 + dx, h0 + dy, n0);
              tma_load_2d(&maps.b8, &full_bar[s], sb, (c.t * chunks + c.ch) * 128, colbase);
              e4m3 = true;
            }
          }
          if (!e4m3) {
            const int kcol = c.base + (c.t * chunks + c.ch) * 64;
            tma_load_4d(&maps.a[c.seg], &full_bar[s], sa, c.ch * 64, w0 + dx, h0 + dy, n0);
            tma_load_2d(&maps.b, &full_bar[s], sb, kcol, colbase);
          }
          if (++c.ch == chunks) {
            c.ch = 0;
            if (++c.t == taps) { c.t = 0; if (!A8 || c.seg != 0) c.base += taps * chunks * 64; ++c.seg; }
          }
          while (c.seg < 3 && p.seg_chunks[c.seg] == 0) ++c.seg;
        }
      }
      // the residual's units as k-blocks nunits, nunits + 1, ...: each goes into its slot as soon as the main loop
      // releases it, so only the last units can arrive after the last wgmma group
      if (p.residual != nullptr) {
        const uint32_t bytes = static_cast<uint32_t>(Cfg::UNIT_BOXES * Cfg::F32_BOX) >> (p.res_up ? 2 : 0);
#pragma unroll 1
        for (int i = 0; i < Cfg::UNITS; ++i) {
          const uint32_t g = static_cast<uint32_t>(nunits + i);
          const int s = static_cast<int>(g % STAGES);
          const int q = SLAB ? s : i;            // SLAB: every slot holds a unit, so unit q stays in slot q
          if (g >= STAGES) mbar_wait(&empty_bar[s], ((g / STAGES) - 1) & 1);
          mbar_arrive_expect_tx(&full_bar[s], bytes);
#pragma unroll
          for (int k = 0; k < Cfg::UNIT_BOXES; ++k)
            tma_load_4d(&maps.r, &full_bar[s], unit_ring + s * Cfg::UNIT_STRIDE + k * Cfg::F32_BOX,
                        colbase + q * Cfg::UNIT_CH + k * Cfg::F32_CH, rw0, rh0, n0);
        }
      }
    }
    return;                                      // the consumers' barriers below count 256 threads
  }

  // ===================================== main loop =====================================
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

  if constexpr (SLAB) {
    // the producer's order; a slab is released once the group of its last k-block has retired, like a weight slot
    const uint32_t row_bytes = static_cast<uint32_t>(p.TW) * 128u;    // one image row of the tile: dy + 1 rows into the slab
    uint32_t u = 0, a = 0;
#pragma unroll 1
    for (int sg = 0; sg < 3; ++sg) {
      const int nx = p.seg_taps[sg] == 9 ? 3 : 1;
      const int loads = p.seg_chunks[sg] * nx;
#pragma unroll 1
      for (int l = 0; l < loads; ++l, ++a) {
        const uint32_t sl = a % SLAB_STAGES;
        mbar_wait(&slab_full[sl], (a / SLAB_STAGES) & 1);
        const uint32_t sa = smem_u32(slab_ring + sl * Cfg::SLAB_BYTES) + wg * 64 * 128;
#pragma unroll 1
        for (int yi = 0; yi < nx; ++yi, ++u) {
          const uint32_t s = u % STAGES;
          mbar_wait(&full_bar[s], (u / STAGES) & 1);
          wgmma_fence();
          const uint64_t da = make_smem_desc_sw128(sa + yi * row_bytes, 1024, 16);
          const uint64_t db = make_smem_desc_sw128(smem_u32(w_ring + s * Cfg::B_BYTES), 1024, 16);
          if (A8 && sg == 0) {                   // warp-uniform
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_ss_e4m3<BN>(acc, da + 2 * k, db + 2 * k, (u | k) != 0 ? 1u : 0u);
          } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_ss<BN>(acc, da + 2 * k, db + 2 * k, (u | k) != 0 ? 1u : 0u);
          }
          wgmma_commit();
          // group u - 1 has retired: its weight slot, and at the first k-block of a load the previous load's slab, go back
          wgmma_wait<1>();
          if (u > 0 && lane == 0) {
            mbar_arrive(&empty_bar[(u - 1) % STAGES]);
            if (yi == 0) mbar_arrive(&slab_empty[(a - 1) % SLAB_STAGES]);
          }
        }
      }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (lane == 0) {
      mbar_arrive(&empty_bar[(u - 1) % STAGES]);
      mbar_arrive(&slab_empty[(a - 1) % SLAB_STAGES]);
    }
  } else {
#pragma unroll 1
    for (int u = 0; u < nunits; ++u) {
      const uint32_t g = static_cast<uint32_t>(u);
      const int s = static_cast<int>(g % STAGES);
      mbar_wait(&full_bar[s], (g / STAGES) & 1);
      const uint32_t sa = smem_u32(smem + s * Cfg::STAGE_BYTES);
      const uint32_t sb = sa + Cfg::A_BYTES;
      wgmma_fence();
      const uint64_t da = make_smem_desc_sw128(sa + wg * 64 * 128, 1024, 16);
      const uint64_t db = make_smem_desc_sw128(sb, 1024, 16);
      if (A8 && u < nunits8) {                     // warp-uniform
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss_e4m3<BN>(acc, da + 2 * k, db + 2 * k, (u | k) != 0 ? 1u : 0u);
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<BN>(acc, da + 2 * k, db + 2 * k, (u | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      // group u stays in flight; group u - 1 has retired, so its slot goes back to the producer
      wgmma_wait<1>();
      if (u > 0 && lane == 0) mbar_arrive(&empty_bar[(g - 1) % STAGES]);
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (lane == 0) mbar_arrive(&empty_bar[static_cast<uint32_t>(nunits - 1) % STAGES]);
  }

  // ===================================== epilogue =====================================
  // Every NHWC value is staged in shared memory (Cfg: fp32 units over the ring, the fp16 tile beside them) and leaves by
  // TMA box stores, which clip at the tensor's extent: the batch tail (n >= N) and the padded columns past Cout are never
  // written.  NCHW (out_mode 2) keeps direct stores.
  const int wr = warp & 3;
  const int quad = lane & 3;
  // Staged addresses are 32-bit shared-window offsets: with the producer warp in the CTA, two CTAs per SM leave 96
  // registers per thread, and the 64 accumulators plus 64-bit addresses would spill.  A box row of RB bytes is swizzled by
  // XOR-ing (row bits) << 4 into its 16-byte chunk index, and the column's byte offset shares no bits with the row's
  // offset, so an element's offset is (row base ^ row swizzle ^ thread column) ^ (column group's bytes).
  constexpr int RB32 = Cfg::F32_CH * 4, RB16 = Cfg::F16_CH * 2;
  const uint32_t s_res = static_cast<uint32_t>(nunits) % STAGES;   // per tap: the stage of unit 0
  auto row_base = [](uint32_t r, int rb) {
    const uint32_t m = rb >= 128 ? 7u : rb == 64 ? 3u : rb == 32 ? 1u : 0u;
    return r * rb ^ ((((r * rb) >> 7) & m) << 4);
  };
  const uint32_t units_u32 = smem_u32(unit_ring);
  auto unit_at = [&](int u) { return units_u32 + (SLAB ? u : (s_res + u) % STAGES) * Cfg::UNIT_STRIDE; };
  // column group j (8 channels) of the thread's pair: unit, box in the unit and the group's bytes in the row
  auto f32_at = [&](int j, uint32_t t) {
    if constexpr (Cfg::F32_CH >= 8) {
      const int cl = 8 * j;
      return unit_at(cl / Cfg::UNIT_CH) + (cl % Cfg::UNIT_CH) / Cfg::F32_CH * Cfg::F32_BOX + (t ^ (cl % Cfg::F32_CH) * 4);
    } else {                                     // 4-channel units (SLAB, BN 16): the pair's unit depends on quad
      return unit_at(2 * j + (quad >> 1)) + t;
    }
  };
  const int rows_per_n = p.TW * p.TH;
  bool ok[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) ok[i] = n0 + (wg * 64 + wr * 16 + (lane >> 2) + 8 * i) / rows_per_n < p.N;

  // bias and residual, into the accumulators
  if (p.residual != nullptr) {
#pragma unroll 1
    for (int q = 0; q < Cfg::UNITS; ++q) {
      const uint32_t g = static_cast<uint32_t>(nunits + q);
      mbar_wait(&full_bar[g % STAGES], (g / STAGES) & 1);
    }
  }
  {
    uint32_t tr[2];                              // residual box row (under res_up the 2x-upsample source row)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = wg * 64 + wr * 16 + (lane >> 2) + 8 * i;
      const int nl = row / rows_per_n, hl = (row / p.TW) % p.TH, xl = row % p.TW;
      const uint32_t rr = p.res_up ? (nl * (p.TH >> 1) + (hl >> 1)) * (p.TW >> 1) + (xl >> 1) : row;
      tr[i] = row_base(rr, RB32) ^ ((8 * quad) % RB32);
    }
    const float* bias = p.bias + colbase + 2 * quad;   // columns < Cout_pad, the bias' extent
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const float2 b = make_float2(__ldg(bias + 8 * j), __ldg(bias + 8 * j + 1));
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float v0, v1;
        if (A8) {
          v0 = fmaf(acc[4 * j + 2 * i], p.acc_scale, b.x); v1 = fmaf(acc[4 * j + 2 * i + 1], p.acc_scale, b.y);
        } else {
          v0 = acc[4 * j + 2 * i] + b.x; v1 = acc[4 * j + 2 * i + 1] + b.y;
        }
        if (p.residual != nullptr) {
          float r0, r1;
          asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];\n" : "=f"(r0), "=f"(r1) : "r"(f32_at(j, tr[i])) : "memory");
          v0 += r0; v1 += r1;
        }
        acc[4 * j + 2 * i] = v0; acc[4 * j + 2 * i + 1] = v1;
      }
    }
  }

  if (p.out_mode == 2) {                         // NCHW: planes of Cout channels, no statistics
    const uint32_t hw = static_cast<uint32_t>(p.H) * p.W;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (!ok[i]) continue;
      const int row = wg * 64 + wr * 16 + (lane >> 2) + 8 * i;
      const int nl = row / rows_per_n, hl = (row / p.TW) % p.TH, xl = row % p.TW;
      float* o = reinterpret_cast<float*>(p.out) + (static_cast<size_t>(n0 + nl) * p.Cout + colbase + 2 * quad) * hw +
                 static_cast<uint32_t>(h0 + hl) * p.W + (w0 + xl);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j, o += 8 * static_cast<size_t>(hw)) {
        const int c = colbase + 8 * j + 2 * quad;
        if (c >= p.Cout) continue;
        o[0] = acc[4 * j + 2 * i];
        if (c + 1 < p.Cout) o[hw] = acc[4 * j + 2 * i + 1];
      }
    }
    return;
  }
  // both warpgroups' last groups have retired (the staging overwrites their operands), and every residual element has been
  // read (under res_up the outputs overwrite source rows that other threads read)
  asm volatile("bar.sync 1, %0;\n" ::"n"(Cfg::CONSUMER_THREADS) : "memory");

  const uint32_t f16_u32 = SLAB ? smem_u32(slab_ring) : smem_u32(smem) + ((s_res + Cfg::UNITS) % STAGES) * Cfg::STAGE_BYTES;
  uint32_t t32[2], t16[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const uint32_t row = wg * 64 + wr * 16 + (lane >> 2) + 8 * i;
    t32[i] = row_base(row, RB32) ^ ((8 * quad) % RB32);
    t16[i] = row_base(row, RB16) ^ (4 * quad);
  }
  const bool do_stats = p.stats != nullptr;
  const int c_left = p.Cout - (colbase + 2 * quad);           // column 8j + 2 quad of the tile is valid while 8j < c_left
  const uint32_t st_u32 = smem_u32(stat_smem) + (warp * 2 * BN + 2 * quad) * 4;   // [warp][sum|sumsq][column]
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
      const uint32_t a16 = f16_u32 + (8 * j) / Cfg::F16_CH * Cfg::F16_BOX + (t16[i] ^ ((8 * j) % Cfg::F16_CH) * 2);
      if (p.out_mode == 0) {
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};\n" ::"r"(f32_at(j, t32[i])), "f"(v0), "f"(v1) : "memory");
        if (p.out16 != nullptr) asm volatile("st.shared.b32 [%0], %1;\n" ::"r"(a16), "r"(pack_h2(v0, v1)) : "memory");
      } else {
        const __half2 hv = __floats2half2_rn(v0, v1);
        asm volatile("st.shared.b32 [%0], %1;\n" ::"r"(a16), "r"(*reinterpret_cast<const uint32_t*>(&hv)) : "memory");
        const float2 r = __half22float2(hv);
        v0 = r.x; v1 = r.y;
      }
      if (ok[i] && 8 * j < c_left) {
        s0 += v0; s1 += v1;
        q0 = fmaf(v0, v0, q0); q1 = fmaf(v1, v1, q1);
      }
    }
    if (do_stats) {
      // column sums over the warp's 16 rows (the 8 lanes that share `quad`); lanes 0..3 keep them
#pragma unroll
      for (int off = 4; off < 32; off <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, off);
        s1 += __shfl_xor_sync(0xffffffffu, s1, off);
        q0 += __shfl_xor_sync(0xffffffffu, q0, off);
        q1 += __shfl_xor_sync(0xffffffffu, q1, off);
      }
      if (lane < 4) {
        const uint32_t st = st_u32 + 32 * j;
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};\n" ::"r"(st), "f"(s0), "f"(s1) : "memory");
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};\n" ::"r"(st + 4 * BN), "f"(q0), "f"(q1) : "memory");
      }
    }
  }
  // the staged tile (and the statistics scratch) is complete: one thread hands the boxes to TMA
  fence_proxy_async_smem();
  asm volatile("bar.sync 1, %0;\n" ::"n"(Cfg::CONSUMER_THREADS) : "memory");
  if (tid == 0) {
    if (p.out_mode == 0) {
#pragma unroll
      for (int q = 0; q < Cfg::UNITS * Cfg::UNIT_BOXES; ++q) {
        const int u = q / Cfg::UNIT_BOXES, k = q % Cfg::UNIT_BOXES;
        const int col = colbase + q * Cfg::F32_CH;
        if (col < p.Cout)
          tma_store_4d(&maps.o, unit_ring + (SLAB ? u : (s_res + u) % STAGES) * Cfg::UNIT_STRIDE + k * Cfg::F32_BOX, col, w0, h0, n0);
      }
    }
    if (p.out_mode == 1 || p.out16 != nullptr) {
#pragma unroll
      for (int q = 0; q < BN / Cfg::F16_CH; ++q) {
        const int col = colbase + q * Cfg::F16_CH;
        if (col < p.Cout) tma_store_4d(&maps.o16, (SLAB ? slab_ring : smem + ((s_res + Cfg::UNITS) % STAGES) * Cfg::STAGE_BYTES) + q * Cfg::F16_BOX, col, w0, h0, n0);
      }
    }
    tma_store_commit();
  }
  if (do_stats) {
    // a warp's 16 rows belong to one sample (TW*TH >= 32); the warps of each sample are combined in a fixed order, so the
    // statistics are reproducible bit for bit, and one fp64 atomic pair per (sample, channel) and tile goes to global memory.
    // They run while the stores are in flight.
    const int n_tile = (128 + rows_per_n - 1) / rows_per_n;
    for (int e = tid; e < n_tile * BN; e += Cfg::CONSUMER_THREADS) {
      const int sn = e / BN, c = e - sn * BN;
      const int n = n0 + sn, col = colbase + c;
      if (n >= p.N || col >= p.Cout) continue;
      float ssum = 0.f, qsum = 0.f;
      for (int w8 = 0; w8 < 8; ++w8) {
        if ((w8 * 16) / rows_per_n != sn) continue;
        ssum += stat_smem[w8 * 2 * BN + c];
        qsum += stat_smem[w8 * 2 * BN + BN + c];
      }
      double* st = p.stats + (static_cast<size_t>(n) * p.Cout + col) * 2;
      atomicAdd(st, static_cast<double>(ssum));
      atomicAdd(st + 1, static_cast<double>(qsum));
    }
  }
  // the shared memory the stores read must outlive them
  if (tid == 0) tma_store_wait_read();
}

}  // namespace ivid
