// Kernel instantiation + host launch wrappers.
#include "ops.h"

#include <algorithm>
#include <cmath>
#include <mutex>

#include "attention.cuh"
#include "attention_hd.cuh"
#include "conv_gemm.cuh"
#include "elementwise.cuh"
#include "embed.cuh"

namespace ivid {

// --------------------------------------------------------------------------------------------------
// conv implicit GEMM
// --------------------------------------------------------------------------------------------------
struct ConvLaunch {
  ConvMaps8 maps;              // b8 is used by the A8 kernels only
  ConvGemmParams p;
  int BN;
  bool a8;
  bool slab;                   // the 3x3 segments load one (TH + 2)-row slab per (chunk, dx): conv_gemm_kernel<BN, A8, true>
  int grid;
};

int conv_pad_cout(int cout) {
  if (cout >= 64) return ((cout + 63) / 64) * 64;
  return ((cout + 15) / 16) * 16;
}
// Pixel tile of the default kernel: TW = the largest power of two <= 16 that divides W, TH = the largest power of two
// <= 128 / TW that divides H, TN = 128 / (TW * TH) samples.  For power-of-two sizes this is min(W, 16) x min(H, 128 / TW);
// for any size the tiles never overhang the image, so only the batch tail is masked.
static int pow2_divisor(int v, int cap) {
  int t = 1;
  while (t * 2 <= cap && v % (t * 2) == 0) t *= 2;
  return t;
}
void conv_tile(int H, int W, int* TW, int* TH, int* TN) {
  IVID_REQUIRE(H > 0 && W > 0, "conv: spatial size must be positive");
  *TW = pow2_divisor(W, 16);
  *TH = pow2_divisor(H, 128 / *TW);
  *TN = 128 / (*TW * *TH);
}
bool conv_can_fuse_stats(int H, int W) {
  int TW, TH, TN;
  conv_tile(H, W, &TW, &TH, &TN);
  return TW * TH >= 32;
}
// 128-wide tiles keep the 64 x 128 fp32 accumulator of a warpgroup at 64 registers per thread, so two CTAs share an SM
int conv_pick_bn(int cout_pad) {
  if (cout_pad % 128 == 0) return 128;
  if (cout_pad % 64 == 0) return 64;
  if (cout_pad % 16 == 0 && cout_pad <= 48) return 16;
  throw Error(kErrInvalidArgument, "conv: unsupported padded Cout " + std::to_string(cout_pad));
}

// The epilogue writes channel pairs (c, c + 1) under c < Cout: an NHWC output of Cout % 8 == 0 channels (the 16-byte row
// pitch of the fp16 tensors that TMA reads next) keeps every pair inside the row and every 4- / 8-byte access aligned.
bool conv_can_res_up(int W, int cout) { return W >= 16 && W % 2 == 0 && cout % 8 == 0; }
bool conv_can_out16(int cout) { return cout % 8 == 0; }
int conv_pad_k(int c) { return ((c + 63) / 64) * 64; }
int conv_pad_k8(int c) { return ((c + 127) / 128) * 128; }
int conv_seg_cols(int taps, int c) { return taps * conv_pad_k(c); }

ConvPack conv_pack(const float* w, const float* b, int cout, int cin, int ksz, int pitch, const float* w2, const float* b2,
                   int cin2, int cin2a, bool e4m3) {
  ConvPack pk;
  const int taps = ksz * ksz;
  pk.cout_pad = conv_pad_cout(cout);
  // e4m3: a power-of-two scale with max|w| * 2^e in (224, 448], shared by the fp16 skip columns
  float scale = 1.f;
  if (e4m3) {
    IVID_REQUIRE(pitch == conv_pad_k(cin), "internal: an e4m3 segment 0 is an ordinary 3x3 or 1x1 conv");
    float mx = 0.f;
    for (size_t i = 0; i < static_cast<size_t>(cout) * cin * taps; ++i) mx = std::max(mx, std::fabs(w[i]));
    const int e = fp8_weight_exponent(mx);
    const float kMinNormal16 = std::ldexp(1.0f, -14);
    if (cin % 16 != 0) pk.refused = "its input channels are not a multiple of 16";
    else if (e < -100 || e > 100) pk.refused = "its weight exponent is outside [-100, 100]";
    for (size_t i = 0; pk.refused == nullptr && i < static_cast<size_t>(cout) * cin2; ++i) {
      const float v = std::fabs(w2[i]), sv = v * std::ldexp(1.0f, e);
      if (sv > 65504.f) pk.refused = "its skip weights times 2^e overflow fp16";
      else if (v >= kMinNormal16 && sv < kMinNormal16) pk.refused = "its skip weights times 2^e become fp16 subnormals";
    }
    pk.e4m3 = pk.refused == nullptr;
    if (pk.e4m3) { pk.e = e; scale = std::ldexp(1.0f, e); }
  }
  const int s0 = cin2a > 0 ? cin2a : cin2, s1 = cin2 - s0;
  const int k0 = pk.e4m3 ? 0 : conv_seg_cols(1, taps * pitch);     // segment 0 padded once, at its end
  pk.K = k0 + conv_seg_cols(1, s0) + conv_seg_cols(1, s1);
  pk.w16.assign(static_cast<size_t>(pk.cout_pad) * pk.K, __float2half_rn(0.f));
  const int cp8 = conv_pad_k8(cin), K8 = pk.e4m3 ? taps * cp8 : 0;
  pk.w8.assign(static_cast<size_t>(pk.cout_pad) * K8, 0);
  for (int co = 0; co < cout; ++co) {
    __half* row = pk.w16.data() + static_cast<size_t>(co) * pk.K;
    for (int tap = 0; tap < taps; ++tap)
      for (int ci = 0; ci < cin; ++ci) {
        const float v = w[(static_cast<size_t>(co) * cin + ci) * taps + tap];
        if (pk.e4m3) pk.w8[static_cast<size_t>(co) * K8 + tap * cp8 + ci] = fp8_e4m3_from_float(v * scale);
        else row[tap * pitch + ci] = __float2half_rn(v);
      }
    for (int ci = 0; ci < cin2; ++ci)
      row[k0 + (ci < s0 ? ci : conv_pad_k(s0) + ci - s0)] = __float2half_rn(w2[static_cast<size_t>(co) * cin2 + ci] * scale);
  }
  pk.bias.assign(pk.cout_pad, 0.f);
  for (int i = 0; i < cout; ++i) {
    if (b != nullptr) pk.bias[i] = b[i];
    if (b2 != nullptr) pk.bias[i] += b2[i];
  }
  return pk;
}

template <int BN, bool SLAB>
static void epilogue_box_channels(int* f32_ch, int* f16_ch) {
  *f32_ch = ConvGemmCfg<BN, SLAB>::F32_CH;
  *f16_ch = ConvGemmCfg<BN, SLAB>::F16_CH;
}
static void epilogue_box_channels(int BN, bool slab, int* f32_ch, int* f16_ch) {
  switch (BN) {
    case 128: slab ? epilogue_box_channels<128, true>(f32_ch, f16_ch) : epilogue_box_channels<128, false>(f32_ch, f16_ch); break;
    case 64: slab ? epilogue_box_channels<64, true>(f32_ch, f16_ch) : epilogue_box_channels<64, false>(f32_ch, f16_ch); break;
    default: slab ? epilogue_box_channels<16, true>(f32_ch, f16_ch) : epilogue_box_channels<16, false>(f32_ch, f16_ch); break;
  }
}

ConvLaunch* conv_launch_create(const ConvDesc& d) {
  IVID_REQUIRE(d.C0 > 0 && d.C0 % 8 == 0, "conv: segment-0 channels must be a positive multiple of 8");
  IVID_REQUIRE(d.C1 % 8 == 0, "conv: segment-1 channels must be a multiple of 8");
  IVID_REQUIRE(d.taps0 == 9 || d.taps0 == 1, "conv: only 3x3 (pad 1) and 1x1 kernels are on this path");
  IVID_REQUIRE(d.taps1 == 9 || d.taps1 == 1, "conv: only 3x3 (pad 1) and 1x1 kernels are on this path");
  IVID_REQUIRE(d.C2 % 8 == 0 && (d.taps2 == 9 || d.taps2 == 1), "conv: segment 2 must be a multiple of 8 channels, 3x3 or 1x1");
  IVID_REQUIRE(d.N > 0 && static_cast<int64_t>(d.N) * d.H * d.W < (int64_t{1} << 31),
               "conv: N*H*W must be below 2^31 (32-bit pixel indices in the epilogue)");
  const bool a8 = d.weight8 != nullptr;
  IVID_REQUIRE(!a8 || d.C0 % 16 == 0, "conv: an e4m3 segment 0 needs a multiple of 16 channels (16-byte TMA rows)");
  auto* l = new ConvLaunch();
  l->a8 = a8;
  ConvGemmParams& p = l->p;
  p.N = d.N; p.H = d.H; p.W = d.W;
  conv_tile(d.H, d.W, &p.TW, &p.TH, &p.TN);
  p.tiles_w = d.W / p.TW;
  p.tiles_h = d.H / p.TH;
  p.tiles_n = (d.N + p.TN - 1) / p.TN;
  // The slab of a 3x3 segment spans TH + 2 rows of one sample, and its one-row shift of TW * 128 bytes must be a whole
  // number of 1024-byte swizzle atoms: tiles of one sample (TN == 1, so TW * TH == 128 and TH + 2 <= 18 rows, within the
  // 256-row TMA box limit) with TW >= 8: 16 x 8 tiles (W % 16 == 0, H % 8 == 0) and 8 x 16 tiles (W % 8 == 0, H % 16 == 0).
  const bool any3x3 = d.taps0 == 9 || (d.C1 > 0 && d.taps1 == 9) || (d.C2 > 0 && d.taps2 == 9);
  l->slab = any3x3 && p.TN == 1 && p.TW >= 8;
  IVID_REQUIRE(!l->slab || p.TW * (p.TH + 2) * 128 <= (ConvGemmCfg<128, true>::SLAB_BYTES), "internal: conv slab larger than its slot");
  l->BN = conv_pick_bn(d.cout_pad);
  p.n_blocks = d.cout_pad / l->BN;
  p.seg_chunks[0] = a8 ? conv_pad_k8(d.C0) / 128 : conv_pad_k(d.C0) / 64; p.seg_taps[0] = d.taps0;
  p.acc_scale = d.acc_scale;
  p.seg_chunks[1] = conv_pad_k(d.C1) / 64; p.seg_taps[1] = d.C1 > 0 ? d.taps1 : 0;
  p.seg_chunks[2] = conv_pad_k(d.C2) / 64; p.seg_taps[2] = d.C2 > 0 ? d.taps2 : 0;
  p.Cout = d.cout; p.ldc = d.ldc; p.ldr = d.ldr; p.out_mode = d.out_mode;
  p.bias = d.bias; p.residual = d.residual; p.out = d.out;
  p.stats = (d.stats != nullptr && conv_can_fuse_stats(d.H, d.W) && d.out_mode != 2) ? d.stats : nullptr;
  IVID_REQUIRE(d.stats == nullptr || p.stats != nullptr, "conv: fused statistics need >= 32 pixels per sample per warp");
  IVID_REQUIRE(d.out_mode == 2 || (d.cout % 8 == 0 && d.ldc % 8 == 0), "conv: NHWC output needs Cout % 8 == 0");
  IVID_REQUIRE(d.residual == nullptr || (d.out_mode != 2 && d.ldr % 4 == 0 && d.ldr >= d.cout),
               "conv: residual needs an NHWC output and a row pitch of >= Cout, a multiple of 4 elements");
  p.res_up = 0;
  if (d.residual != nullptr && d.residual_up) {
    IVID_REQUIRE(conv_can_res_up(d.W, d.cout) && d.H % 2 == 0, "conv: upsampled residual needs an even W >= 16 and Cout % 8 == 0");
    p.res_up = 1;
  }
  // the epilogue's TMA boxes: 16-byte aligned tensors
  auto aligned = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; };
  IVID_REQUIRE(d.out_mode == 2 || (aligned(d.out) && aligned(d.out16) && aligned(d.residual)),
               "conv: NHWC output, fp16 copy and residual must be 16-byte aligned");
  p.out16 = nullptr;
  if (d.out16 != nullptr) {
    IVID_REQUIRE(d.out_mode == 0 && conv_can_out16(d.cout), "conv: fp16 output copy needs an fp32 NHWC output and Cout % 8 == 0");
    p.out16 = static_cast<__half*>(d.out16);
  }
  // packed weight columns: every segment padded to whole 64-channel chunks per tap (zero columns); the activation maps keep
  // the real channel extent, so TMA zero-fills the missing channels of a segment's last chunk
  // (fp8 mode: segment 0's columns live in weight8, so the fp16 matrix holds the skip segments only)
  const int Ktot = (a8 ? 0 : conv_seg_cols(d.taps0, d.C0)) + conv_seg_cols(d.taps1, d.C1) + conv_seg_cols(d.taps2, d.C2);
  ConvMaps8& M = l->maps;
  // a slab segment's box is TH + 2 rows, loaded from row h0 - 1 (TMA zero-fills the halo rows outside the image)
  auto rows = [&](int taps) { return l->slab && taps == 9 ? p.TH + 2 : p.TH; };
  M.a[0] = a8 ? make_act_map(d.act0, d.N, d.H, d.W, d.C0, p.TW, rows(d.taps0), p.TN, CU_TENSOR_MAP_DATA_TYPE_UINT8)
              : make_act_map(d.act0, d.N, d.H, d.W, d.C0, p.TW, rows(d.taps0), p.TN);
  M.a[1] = d.C1 > 0 ? make_act_map(d.act1, d.N, d.H, d.W, d.C1, p.TW, rows(d.taps1), p.TN) : M.a[0];
  M.a[2] = d.C2 > 0 ? make_act_map(d.act2, d.N, d.H, d.W, d.C2, p.TW, rows(d.taps2), p.TN) : M.a[0];
  if (a8) {
    M.b8 = make_weight_map(d.weight8, d.cout_pad, d.taps0 * conv_pad_k8(d.C0), l->BN, CU_TENSOR_MAP_DATA_TYPE_UINT8);
    M.b = Ktot > 0 ? make_weight_map(d.weight, d.cout_pad, Ktot, l->BN) : M.b8;    // no skip segment: b is never read
  } else {
    M.b = make_weight_map(d.weight, d.cout_pad, Ktot, l->BN);
  }
  // epilogue: fp32 boxes of F32_CH channels and fp16 boxes of F16_CH, as the kernel stages them (ConvGemmCfg)
  int f32_ch = 0, f16_ch = 0;
  epilogue_box_channels(l->BN, l->slab, &f32_ch, &f16_ch);
  const auto f32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  M.r = M.o = M.o16 = M.a[0];                                     // placeholders of the maps a launch does not read
  if (d.residual != nullptr) {
    const int up = p.res_up ? 1 : 0;
    M.r = make_act_map(d.residual, d.N, d.H >> up, d.W >> up, d.cout, p.TW >> up, p.TH >> up, p.TN, f32, d.ldr, f32_ch);
  }
  if (d.out_mode == 0) M.o = make_act_map(d.out, d.N, d.H, d.W, d.cout, p.TW, p.TH, p.TN, f32, d.ldc, f32_ch);
  const void* o16 = d.out_mode == 1 ? d.out : d.out_mode == 0 ? d.out16 : nullptr;
  if (o16 != nullptr) M.o16 = make_act_map(o16, d.N, d.H, d.W, d.cout, p.TW, p.TH, p.TN, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, d.ldc, f16_ch);
  l->grid = p.tiles_w * p.tiles_h * p.tiles_n * p.n_blocks;     // one CTA per (pixel tile, column block)
  return l;
}
void conv_launch_destroy(ConvLaunch* l) { delete l; }
int conv_launch_bn(const ConvLaunch* l) { return l->BN; }
bool conv_launch_a8(const ConvLaunch* l) { return l->a8; }

template <int BN, bool A8, bool SLAB>
static void run_conv(const ConvLaunch* l, cudaStream_t s) {
  using Cfg = ConvGemmCfg<BN, SLAB>;
  static std::once_flag once;
  std::call_once(once, [] {
    IVID_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<BN, A8, SLAB>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  });
  if constexpr (A8) conv_gemm_kernel<BN, true, SLAB><<<l->grid, Cfg::THREADS, Cfg::SMEM_BYTES, s>>>(l->maps, l->p);
  else conv_gemm_kernel<BN, false, SLAB><<<l->grid, Cfg::THREADS, Cfg::SMEM_BYTES, s>>>(static_cast<const ConvMaps&>(l->maps), l->p);
  IVID_CHECK_CUDA(cudaGetLastError());
}
template <bool A8, bool SLAB>
static void run_conv_bn(const ConvLaunch* l, cudaStream_t s) {
  switch (l->BN) {
    case 128: run_conv<128, A8, SLAB>(l, s); break;
    case 64: run_conv<64, A8, SLAB>(l, s); break;
    default: run_conv<16, A8, SLAB>(l, s); break;
  }
}
void conv_launch_run_out(const ConvLaunch* l, void* out, cudaStream_t s) {
  IVID_REQUIRE(l->p.out_mode == 2, "internal: only an NCHW conv output is patched at run time (NHWC outputs are in tensor maps)");
  ConvLaunch tmp = *l;
  tmp.p.out = out;
  conv_launch_run(&tmp, s);
}
void conv_launch_run(const ConvLaunch* l, cudaStream_t s) {
  if (l->a8) {
    if (l->slab) run_conv_bn<true, true>(l, s);
    else run_conv_bn<true, false>(l, s);
  } else {
    if (l->slab) run_conv_bn<false, true>(l, s);
    else run_conv_bn<false, false>(l, s);
  }
}

static int ew_grid(size_t work_items, int block) {
  const size_t blocks = (work_items + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count()) * 16;
  return static_cast<int>(std::max<size_t>(1, std::min(blocks, cap)));
}

// --------------------------------------------------------------------------------------------------
// attention
// --------------------------------------------------------------------------------------------------
struct AttnLaunch {
  CUtensorMap mapQ, mapKV;
  AttnParams p;          // head width 64: attention_kernel
  AttnHdParams hp;       // other widths: attention_hd_kernel<nv, qres>
  int head_ch = 64;
  int nv = 0;
  bool qres = false;
  int smem = 0;
  int grid;
  // rows [row0, N) take the identity output (attention_identity_kernel); the softmax kernels run over rows [0, row0)
  int N = 0, T = 0, C = 0, row0 = 0;
  const __half* qkv = nullptr;
  __half* out = nullptr;
};

AttnLaunch* attn_launch_create(const void* qkv, int N, int T, int C, int head_ch, void* out, int row0) {
  if (head_ch <= 0 || head_ch % 64 != 0)
    throw Error(kErrNotImplemented, "attention: head width " + std::to_string(head_ch) + " is not a multiple of 64");
  IVID_REQUIRE(C % head_ch == 0, "attention: channels must be a multiple of the head width " + std::to_string(head_ch));
  IVID_REQUIRE(T >= 1, "attention: sequence length must be positive");
  if (row0 < 0) row0 = N;
  IVID_REQUIRE(row0 <= N, "attention: the perturbed-row start must lie in [0, N]");
  auto* l = new AttnLaunch();
  l->N = N; l->T = T; l->C = C; l->row0 = row0;
  l->qkv = static_cast<const __half*>(qkv);
  l->out = static_cast<__half*>(out);
  l->head_ch = head_ch;
  l->p.N = N; l->p.T = T; l->p.C = C; l->p.heads = C / 64;
  l->p.q_tiles = (T + 127) / 128;
  l->p.out = reinterpret_cast<__half*>(out);
  const uint64_t dims[3] = {static_cast<uint64_t>(3 * C), static_cast<uint64_t>(T), static_cast<uint64_t>(N)};
  const uint64_t str[2] = {static_cast<uint64_t>(3 * C) * 2, static_cast<uint64_t>(T) * 3 * C * 2};
  const uint32_t boxq[3] = {64, 128, 1};
  const uint32_t boxkv[3] = {64, AttnCfg::KV, 1};
  l->mapQ = make_tensor_map(CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(qkv), dims, str, boxq,
                            CU_TENSOR_MAP_SWIZZLE_128B);
  l->mapKV = make_tensor_map(CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(qkv), dims, str, boxkv,
                             CU_TENSOR_MAP_SWIZZLE_128B);
  l->grid = row0 * l->p.heads * l->p.q_tiles;
  if (head_ch == 64) return l;
  // wider heads: k = d/64 chunks; ceil(k/4) output-column slices of nv <= 4 boxes (see attention_hd.cuh)
  using Cfg = AttnHdCfg;
  const int k = head_ch / 64;
  const int slices = (k + 3) / 4;
  l->nv = (k + slices - 1) / slices;
  l->qres = k <= Cfg::RESIDENT_Q_MAX_CHUNKS;
  AttnHdParams& hp = l->hp;
  hp.N = N; hp.T = T; hp.C = C; hp.d = head_ch; hp.heads = C / head_ch; hp.chunks = k;
  hp.q_tiles = l->p.q_tiles;
  hp.slices = (k + l->nv - 1) / l->nv;          // every slice holds >= 1 box
  hp.scale_log2 = static_cast<float>(1.4426950408889634 / std::sqrt(static_cast<double>(head_ch)));
  hp.out = l->p.out;
  const int q_bytes = l->qres ? k * Cfg::QCHUNK_BYTES : 0;
  const int fixed = q_bytes + 1024 /*barriers*/ + 1024 /*align*/;
  const int budget = l->nv == 2 ? Cfg::MAX_SMEM_2CTA : Cfg::MAX_SMEM;
  hp.stages = std::min(Cfg::MAX_STAGES, (budget - fixed) / Cfg::stage_bytes(l->qres));
  IVID_REQUIRE(hp.stages >= 4, "attention: shared-memory ring too shallow");
  l->smem = fixed + hp.stages * Cfg::stage_bytes(l->qres);
  l->grid = row0 * hp.heads * hp.q_tiles * hp.slices;
  return l;
}
void attn_launch_destroy(AttnLaunch* l) { delete l; }

template <int NV, bool QRES>
static void run_attn_hd(const AttnLaunch* l, cudaStream_t s) {
  static std::once_flag once;
  std::call_once(once, [] {
    IVID_CHECK_CUDA(cudaFuncSetAttribute(attention_hd_kernel<NV, QRES>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnHdCfg::MAX_SMEM));
  });
  attention_hd_kernel<NV, QRES><<<l->grid, AttnHdCfg::THREADS, l->smem, s>>>(l->mapQ, l->mapKV, l->hp);
  IVID_CHECK_CUDA(cudaGetLastError());
}

void attn_launch_run(const AttnLaunch* l, cudaStream_t s) {
  attn_launch_run_identity(l, s);
  attn_launch_run_softmax(l, s);
}
void attn_launch_run_identity(const AttnLaunch* l, cudaStream_t s) {
  if (l->row0 == l->N) return;
  const size_t rows = static_cast<size_t>(l->N - l->row0) * l->T;
  attention_identity_kernel<<<ew_grid(rows * (l->C / 8), 256), 256, 0, s>>>(l->qkv, l->out, static_cast<size_t>(l->row0) * l->T, rows,
                                                                         l->C, l->head_ch);
  IVID_CHECK_CUDA(cudaGetLastError());
}
void attn_launch_run_softmax(const AttnLaunch* l, cudaStream_t s) {
  if (l->row0 == 0) return;
  if (l->head_ch != 64) {
    switch (l->nv * 2 + (l->qres ? 1 : 0)) {
      case 5: run_attn_hd<2, true>(l, s); break;
      case 7: run_attn_hd<3, true>(l, s); break;
      case 9: run_attn_hd<4, true>(l, s); break;
      // nv = 2 only at k <= 4 chunks, where Q is always resident: there is no <2, false>
      case 6: run_attn_hd<3, false>(l, s); break;
      case 8: run_attn_hd<4, false>(l, s); break;
      default: throw Error(kErrState, "internal: attention slice width " + std::to_string(l->nv));
    }
    return;
  }
  static std::once_flag once;
  std::call_once(once, [] {
    IVID_CHECK_CUDA(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnCfg::SMEM_BYTES));
  });
  attention_kernel<<<l->grid, AttnCfg::THREADS, AttnCfg::SMEM_BYTES, s>>>(l->mapQ, l->mapKV, l->p);
  IVID_CHECK_CUDA(cudaGetLastError());
}

// --------------------------------------------------------------------------------------------------
// element-wise / embedding
// --------------------------------------------------------------------------------------------------

void launch_gn_stats(const float* x, double* stats, int N, int HW, int C, cudaStream_t s) {
  IVID_REQUIRE(C % 4 == 0, "gn_stats: C % 4");
  dim3 grid((HW + kStatsPixPerBlock - 1) / kStatsPixPerBlock, N);
  gn_stats_kernel<<<grid, 256, 0, s>>>(x, stats, HW, C);
  IVID_CHECK_CUDA(cudaGetLastError());
}

void launch_gn_apply(const GnApplyDesc& d, cudaStream_t s) {
  IVID_REQUIRE(d.C0 % 8 == 0 && d.C1 % 8 == 0, "gn_apply: channel counts must be multiples of 8");
  const int C = d.C0 + d.C1;
  IVID_REQUIRE(d.groups >= 1 && d.groups <= 64 && C % d.groups == 0, "group norm: groups must divide channels (<= 64 groups)");
  IVID_REQUIRE(d.stats0 != nullptr && d.gamma != nullptr && d.beta != nullptr, "gn_apply: statistics / affine parameters missing");
  GnApplyParams p;
  p.x0 = static_cast<const float*>(d.x0); p.x1 = static_cast<const float*>(d.x1); p.C0 = d.C0; p.C1 = d.C1; p.N = d.N; p.H = d.H; p.W = d.W; p.mode = d.mode;
  p.x0h = d.x0_half ? reinterpret_cast<const __half*>(d.x0) : nullptr;
  p.x1h = d.x0_half ? reinterpret_cast<const __half*>(d.x1) : nullptr;
  p.silu = d.silu ? 1 : 0;
  p.stats0 = d.stats0; p.stats1 = d.stats1; p.groups = d.groups; p.inv_count = 1.0 / (static_cast<double>(d.H) * d.W);
  p.eps = d.eps; p.gamma = d.gamma; p.beta = d.beta; p.film = d.film; p.film_ld = d.film_ld; p.film_off = d.film_off;
  p.film_add = d.film_add ? 1 : 0;
  p.out_act = reinterpret_cast<__half*>(d.out_act); p.out_raw16 = reinterpret_cast<__half*>(d.out_raw16);
  p.out_act8 = d.out_e4m3 ? reinterpret_cast<uint8_t*>(d.out_act) : nullptr;
  p.out_raw32 = d.out_raw32;
  p.out_lo = reinterpret_cast<__half*>(d.out_lo);
  IVID_REQUIRE(d.out_lo == nullptr || (d.mode == 0 && d.x0_half && d.out_raw16 == nullptr && d.out_raw32 == nullptr),
               "gn_apply: the split (hi/lo) output exists on the same-resolution fp16-source path only");
  IVID_REQUIRE(!d.out_e4m3 || (d.out_lo == nullptr && C % 16 == 0), "gn_apply: an e4m3 output needs C % 16 == 0 and no split output");
  const int Ho = d.mode == 1 ? d.H * 2 : (d.mode == 2 ? d.H / 2 : d.H);
  const int Wo = d.mode == 1 ? d.W * 2 : (d.mode == 2 ? d.W / 2 : d.W);
  // One wave of blocks (3 resident per SM) split evenly over the samples, so the statistics -> coefficient prologue is
  // paid once per ~1/13th of an image; small tensors still spread over all SMs (>= 1K work items per block).
  {
    const int blocks_per_n = std::max(1, (sm_count() * 3) / std::max(d.N, 1));
    const int by_wave = (Ho * Wo + blocks_per_n - 1) / blocks_per_n;
    const int small = std::max(1, 1024 / (C / 8));      // at least ~4 work items per thread
    p.pix_per_block = std::max(1, std::min(Ho * Wo, std::max(by_wave, small)));
  }
  // the upsampling path walks SOURCE pixels (each written to its 2x2 outputs)
  int pix_space = Ho * Wo;
  if (d.mode == 1) {
    pix_space = d.H * d.W;
    p.pix_per_block = std::max(1, (p.pix_per_block + 3) / 4);
  }
  dim3 grid((pix_space + p.pix_per_block - 1) / p.pix_per_block, d.N);
  const size_t smem = static_cast<size_t>(C) * 8;
  if (p.mode == 0 && p.x0h != nullptr && p.out_raw16 == nullptr && p.out_raw32 == nullptr) {
    const bool hoist = 256 % (C / 8) == 0;
    if (p.out_lo != nullptr) {        // output head only: also emits the low half of the two-term split
      if (hoist) gn_apply_h16_kernel<true, true><<<grid, 256, smem, s>>>(p);
      else gn_apply_h16_kernel<false, true><<<grid, 256, smem, s>>>(p);
    } else if (d.out_e4m3) {
      if (hoist) gn_apply_h16_kernel<true, false, true><<<grid, 256, smem, s>>>(p);
      else gn_apply_h16_kernel<false, false, true><<<grid, 256, smem, s>>>(p);
    } else if (hoist) gn_apply_h16_kernel<true><<<grid, 256, smem, s>>>(p);
    else gn_apply_h16_kernel<false><<<grid, 256, smem, s>>>(p);
  } else if (d.out_e4m3) {
    gn_apply_kernel<true><<<grid, 256, smem, s>>>(p);
  } else {
    gn_apply_kernel<><<<grid, 256, smem, s>>>(p);
  }
  IVID_CHECK_CUDA(cudaGetLastError());
}
void launch_im2col_s2(const void* x16, void* col, int N, int H, int W, int C, cudaStream_t s) {
  IVID_REQUIRE(C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "im2col_s2: C % 8, even spatial size");
  const size_t items = static_cast<size_t>(N) * (H / 2) * (W / 2) * 9 * (C / 8);
  im2col_s2_h16_kernel<<<ew_grid(items, 256), 256, 0, s>>>(reinterpret_cast<const __half*>(x16), reinterpret_cast<__half*>(col), N, H, W, C);
  IVID_CHECK_CUDA(cudaGetLastError());
}
void launch_upsample2x_h16(const void* x16, void* out, int N, int H, int W, int C, cudaStream_t s) {
  IVID_REQUIRE(C % 8 == 0, "upsample2x: C % 8");
  const size_t items = static_cast<size_t>(N) * H * W * 4 * (C / 8);
  upsample2x_h16_kernel<<<ew_grid(items, 256), 256, 0, s>>>(reinterpret_cast<const __half*>(x16), reinterpret_cast<__half*>(out), N, H, W, C);
  IVID_CHECK_CUDA(cudaGetLastError());
}
void launch_resample_f32(const float* x, float* out, void* out16, int N, int H, int W, int C, int mode, cudaStream_t s) {
  IVID_REQUIRE(C % 4 == 0 && (mode == 1 || (H % 2 == 0 && W % 2 == 0)), "resample_f32: C % 4, even spatial size for pooling");
  const size_t items = static_cast<size_t>(N) * (mode == 1 ? 4 * H * W : (H / 2) * (W / 2)) * (C / 4);
  resample_f32_kernel<<<ew_grid(items, 256), 256, 0, s>>>(x, out, reinterpret_cast<__half*>(out16), N, H, W, C, mode);
  IVID_CHECK_CUDA(cudaGetLastError());
}
void launch_pack_input(const float* x, void* out, int N, int Nx, int Cin, int HW, cudaStream_t s) {
  IVID_REQUIRE(Cin >= 1 && Cin <= 16, "pack_input: 1..16 input channels (two-term split inside 64 operand channels)");
  pack_input_kernel<<<ew_grid(static_cast<size_t>(N) * HW, 256), 256, 0, s>>>(x, reinterpret_cast<__half*>(out), N, Nx,
                                                                                 Cin, HW);
  IVID_CHECK_CUDA(cudaGetLastError());
}

void launch_eps_gather(const float* Y, const float* bias, float* eps, int N, int H, int W, int Co, int ldy, cudaStream_t s) {
  IVID_REQUIRE(Co >= 1 && Co <= 7 && 9 * Co <= ldy, "eps_gather: 9*Co tap columns must fit the row pitch");
  IVID_REQUIRE(Co != 4 || ldy % 4 == 0, "eps_gather: row pitch must keep float4 alignment");
  eps_gather_kernel<<<ew_grid(static_cast<size_t>(N) * H * W, 256), 256, 0, s>>>(Y, bias, eps, N, H, W, Co, ldy);
  IVID_CHECK_CUDA(cudaGetLastError());
}

void launch_posenc(const int64_t* t, int Nt, const float* freqs, int half, float* out, int N, cudaStream_t s) {
  posenc_kernel<<<N, 128, 0, s>>>(t, Nt, freqs, half, out, N);
  IVID_CHECK_CUDA(cudaGetLastError());
}

void launch_film_table(const float* emb, const float* Wp, const float* bias, float* x_t, float* out, int N, int K, int O, cudaStream_t s) {
  IVID_REQUIRE(K % 32 == 0 && O % 4 == 0, "film table: K % 32 == 0");
  static std::once_flag once;
  std::call_once(once, [] {
    IVID_CHECK_CUDA(cudaFuncSetAttribute(film_table_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FilmCfg::SMEM_BYTES));
  });
  const int nblk = (N + 31) / 32;
  silu_transpose_kernel<<<std::min(256, (nblk * K * 32 + 255) / 256), 256, 0, s>>>(emb, x_t, N, K, 1);
  const int tiles = (O + FilmCfg::TO - 1) / FilmCfg::TO;
  dim3 grid(std::min(tiles, std::max(1, sm_count() / nblk)), nblk);
  film_table_kernel<<<grid, FilmCfg::THREADS, FilmCfg::SMEM_BYTES, s>>>(Wp, x_t, bias, out, N, K, O);
  IVID_CHECK_CUDA(cudaGetLastError());
}

void launch_linear(const float* in, const float* W, const float* bias, float* out, int N, int K, int O, int silu_in,
                   const float* label_emb, const int64_t* classes, int Ncls, cudaStream_t s) {
  if ((K == 256 || K == 512 || K == 1024) && O <= 8192) {
    dim3 grid((O + 7) / 8, (N + 31) / 32);
    const size_t smem = static_cast<size_t>(32) * K * 4;
    static std::once_flag once;
    std::call_once(once, [] {
      IVID_CHECK_CUDA(cudaFuncSetAttribute(linear_warp_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * 256 * 4));
      IVID_CHECK_CUDA(cudaFuncSetAttribute(linear_warp_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * 512 * 4));
      IVID_CHECK_CUDA(cudaFuncSetAttribute(linear_warp_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * 1024 * 4));
    });
    auto go = [&](auto kern) { kern<<<grid, 256, smem, s>>>(in, W, bias, out, N, O, silu_in, label_emb, classes, Ncls); };
    if (K == 256) go(linear_warp_kernel<2>); else if (K == 512) go(linear_warp_kernel<4>); else go(linear_warp_kernel<8>);
    IVID_CHECK_CUDA(cudaGetLastError());
    return;
  }
  if (K % 32 == 0) {
    if (O >= 128 * 64) {
      dim3 grid((O + 127) / 128, (N + 31) / 32);
      linear_tiled_kernel<4><<<grid, 256, 0, s>>>(in, W, bias, out, N, K, O, silu_in, label_emb, classes, Ncls);
    } else {
      dim3 grid((O + 63) / 64, (N + 31) / 32);
      linear_tiled_kernel<2><<<grid, 256, 0, s>>>(in, W, bias, out, N, K, O, silu_in, label_emb, classes, Ncls);
    }
    IVID_CHECK_CUDA(cudaGetLastError());
    return;
  }
  dim3 grid((O + 63) / 64, (N + 31) / 32);
  linear_rows_kernel<<<grid, 256, 0, s>>>(in, W, bias, out, N, K, O, silu_in, label_emb, classes, Ncls);
  IVID_CHECK_CUDA(cudaGetLastError());
}

}  // namespace ivid
