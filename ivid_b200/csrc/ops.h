// Host-side launch descriptors for the sm_90a kernels (built once at plan time, replayed every step).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "host_util.h"

namespace ivid {

// mirrors of the device parameter structs (defined in the .cuh files; redeclared opaque here through includes in ops.cu)
struct ConvLaunch;
struct AttnLaunch;

struct ConvDesc {
  const void* act0 = nullptr; int C0 = 0; int taps0 = 9;   // segment 0: fp16 NHWC activation, 9 = 3x3, 1 = 1x1
  const void* act1 = nullptr; int C1 = 0; int taps1 = 1;   // optional segment 1 (1x1 skip over another tensor)
  const void* act2 = nullptr; int C2 = 0; int taps2 = 1;   // optional segment 2 (second half of a virtual concat)
  void* out16 = nullptr;                                   // optional fp16 NHWC copy of an fp32 output (same ldc)
  // weights and bias as conv_pack writes them (the stem and the split output head write their own columns in this layout)
  const void* weight = nullptr;                            // fp16 [cout_pad][Ktot], Ktot = sum of conv_seg_cols over segments
  // fp8 operand mode: act0 is e4m3 NHWC (C0 % 16 == 0) and weight8 its e4m3 weights [cout_pad][taps0*conv_pad_k8(C0)],
  // scaled by 2^e; `weight` then holds only the skip segments' columns (fp16, scaled by the same 2^e; null without skip
  // segments), and acc_scale = 2^-e
  const void* weight8 = nullptr;
  float acc_scale = 1.f;
  int cout_pad = 0;
  int cout = 0;                                            // valid output channels
  const float* bias = nullptr;                             // [cout_pad]
  const float* residual = nullptr; int ldr = 0;            // fp32 NHWC
  bool residual_up = false;                                // residual is [N][H/2][W/2][ldr]: added through a nearest-2x upsample (conv_can_res_up)
  void* out = nullptr; int ldc = 0; int out_mode = 0;      // 0 fp32 NHWC, 1 fp16 NHWC, 2 fp32 NCHW
  double* stats = nullptr;                                 // optional fused GroupNorm statistics of the output [N][cout][2]
  int N = 0, H = 0, W = 0;
};

// opaque, heap-allocated launch records (hold the CUtensorMaps)
ConvLaunch* conv_launch_create(const ConvDesc& d);
void conv_launch_destroy(ConvLaunch* l);
void conv_launch_run(const ConvLaunch* l, cudaStream_t s);
int conv_launch_bn(const ConvLaunch* l);
bool conv_launch_a8(const ConvLaunch* l);                  // segment 0 runs as e4m3 (ConvDesc::weight8)
void conv_launch_run_out(const ConvLaunch* l, void* out, cudaStream_t s);   // same launch, output pointer overridden
int conv_pick_bn(int cout_pad);
// whether a conv with this many (unpadded) output channels can also emit the fp16 copy of its fp32 NHWC output
bool conv_can_out16(int cout);
// whether the conv epilogue can add a half-resolution residual through a nearest-2x upsample (output width W, Cout)
bool conv_can_res_up(int W, int cout);
// pixel tile TW x TH x TN (== 128) of the default conv kernel at an H x W layer (see ops.cu)
void conv_tile(int H, int W, int* TW, int* TH, int* TN);
bool conv_can_fuse_stats(int H, int W);                    // epilogue statistics need >= 32 pixels of one sample per warp
int conv_pad_cout(int cout);
// packed weight columns per tap of a K segment of c channels (c % 8 == 0): whole 64-channel chunks, zero columns at the pad
int conv_pad_k(int c);
// the same for an e4m3 segment 0 (c % 16 == 0): whole 128-channel chunks
int conv_pad_k8(int c);
// fp16 weight columns of a K segment of c channels over `taps` taps (0 for c == 0)
int conv_seg_cols(int taps, int c);

// Host-packed operands of one conv, in the layout conv_launch_create reads.
struct ConvPack {
  std::vector<__half> w16;     // [cout_pad][K]: segment 0 (unless e4m3), then the 1x1 skip segments
  std::vector<uint8_t> w8;     // e4m3 only: segment 0 as e4m3(w * 2^e), [cout_pad][taps * conv_pad_k8(cin)]
  std::vector<float> bias;     // [cout_pad]: b + b2
  int cout_pad = 0, K = 0;     // K == 0: an e4m3 conv without skip segments (no fp16 columns)
  bool e4m3 = false;
  int e = 0;                   // weight exponent of an e4m3 segment 0 (0 otherwise); the skip columns hold fp16(w2 * 2^e)
  const char* refused = nullptr;   // why an e4m3 segment 0 was requested but not packed (everything is fp16 then)
};
// Packs w [cout][cin][ksz][ksz] (+ bias b; null: zero) as segment 0 at `pitch` columns per tap: conv_pad_k(cin) for an
// ordinary conv, 64 for the stem, cin for the im2col stride-2 conv (whose taps * cin columns are padded once at the end).
// An optional 1x1 skip conv w2 [cout][cin2] follows as one K segment per part of a concatenated input (the first cin2a
// channels, then the rest; cin2a = 0: one segment); its bias b2 (if not null) is folded into the bias.
// e4m3 asks for segment 0 in e4m3 (DESIGN.md §2), which is refused, leaving the conv fp16, when cin % 16 != 0, when
// |e| > 100, or when a scaled skip weight would overflow fp16 or turn a normal fp16 weight into a subnormal.
ConvPack conv_pack(const float* w, const float* b, int cout, int cin, int ksz, int pitch, const float* w2, const float* b2,
                   int cin2, int cin2a, bool e4m3);

// head_ch = 64: attention_kernel; any other multiple of 64: attention_hd_kernel (kErrNotImplemented otherwise).
// row0 in [0, N] (-1: N): rows [0, row0) run that kernel, exactly as a launch over those rows alone; rows [row0, N) take the
// perturbed-attention identity output, each head's V channels (attention_identity_kernel)
AttnLaunch* attn_launch_create(const void* qkv, int N, int T, int C, int head_ch, void* out, int row0 = -1);
void attn_launch_destroy(AttnLaunch* l);
void attn_launch_run(const AttnLaunch* l, cudaStream_t s);                    // both parts below
void attn_launch_run_softmax(const AttnLaunch* l, cudaStream_t s);            // rows [0, row0) only (nothing at row0 = 0)
void attn_launch_run_identity(const AttnLaunch* l, cudaStream_t s);           // rows [row0, N) only (nothing at row0 = N)

void launch_gn_stats(const float* x, double* stats, int N, int HW, int C, cudaStream_t s);
struct GnApplyDesc {
  const void* x0 = nullptr; const void* x1 = nullptr; int C0 = 0, C1 = 0;
  bool x0_half = false;                                            // sources point at fp16 data (both, when concatenated)
  int N = 0, H = 0, W = 0; int mode = 0; int silu = 1;
  const double* stats0 = nullptr; const double* stats1 = nullptr;   // per-(sample, channel) sum / sumsq of each source
  int groups = 32; float eps = 1e-5f;
  const float* gamma = nullptr; const float* beta = nullptr;        // [C0 + C1]
  const float* film = nullptr; int film_ld = 0, film_off = 0;       // optional FiLM table (scale | shift)
  bool film_add = false;                                            // table holds ONE row per channel, added before the norm
  void* out_act = nullptr; void* out_raw16 = nullptr; float* out_raw32 = nullptr;
  void* out_lo = nullptr;      // optional low half of a two-term fp16 split of the output (fp16-source same-resolution path only)
  bool out_e4m3 = false;       // out_act is e4m3 (one byte per element, satfinite round-to-nearest-even) instead of fp16
};
void launch_gn_apply(const GnApplyDesc& d, cudaStream_t s);
// eps[n][c][h][w] = bias[c] + sum_tap Y[n][h+dy][w+dx][tap*Co + c]  (output head, see eps_gather_kernel)
void launch_eps_gather(const float* Y, const float* bias, float* eps, int N, int H, int W, int Co, int ldy, cudaStream_t s);
// plain Downsample2d / Upsample2d layers (resblock_updown=False): see elementwise.cuh
void launch_im2col_s2(const void* x16, void* col, int N, int H, int W, int C, cudaStream_t s);
void launch_upsample2x_h16(const void* x16, void* out, int N, int H, int W, int C, cudaStream_t s);
void launch_resample_f32(const float* x, float* out, void* out16, int N, int H, int W, int C, int mode, cudaStream_t s);
void launch_pack_input(const float* x, void* out, int N, int Nx, int Cin, int HW, cudaStream_t s);

struct CondPackDesc {
  const float* x = nullptr; const float* y = nullptr; const float* mask = nullptr; const float* mask_rgb = nullptr;
  const float* noise = nullptr; void* out = nullptr; int N = 0, Nx = 0, H = 0, W = 0; int kind = 0;
  int scale = 2;                                            // kind 2: y is [Nx][4][H/scale][W/scale]
  uint64_t seed = 0; uint32_t stream = 0; const int* stream_dev = nullptr;
};
void launch_cond_pack(const CondPackDesc& d, cudaStream_t s);   // sampler.cu
void launch_cfg_mix(const float* eps2, float* out, size_t count, float strength, cudaStream_t s);   // sampler.cu
// the step's guidance mix over row blocks of `count` elements (include/ivid_b200.h, ivid_guidance_mix)   // sampler.cu
void launch_guidance_mix(const float* eps, float* out, size_t count, int cfg, float strength, int pag, float pag_scale,
                         cudaStream_t s);
// dynamic thresholding of x [N][M] (sampler.cuh): s_out [N] and x_out = clamp(x, -s, s) / s; threshold_max <= 0: no upper bound
void launch_dynamic_threshold(const float* x, int N, int M, double ratio, double threshold_max, float* s_out, float* x_out,
                              cudaStream_t s);   // sampler.cu
// adaptive projected guidance of x_0 rows [N][M] (include/ivid_b200.h, ivid_op_apg): state holds m_prev on entry and m on return
void launch_apg(const float* dc, const float* du, float* state, int N, int M, float s, double eta, double norm, double beta,
                float* out, cudaStream_t st);   // sampler.cu

void launch_posenc(const int64_t* t, int Nt, const float* freqs, int half, float* out, int N, cudaStream_t s);
// FiLM table (all ResBlock emb_layers as one product): out = silu(emb) * Wp^T + bias, Wp in the swizzled K-chunk-major
// layout described at film_table_kernel; x_t is a [ceil(N/32)][K][32] fp32 scratch.
void launch_film_table(const float* emb, const float* Wp, const float* bias, float* x_t, float* out, int N, int K, int O, cudaStream_t s);
void launch_linear(const float* in, const float* W, const float* bias, float* out, int N, int K, int O, int silu_in,
                   const float* label_emb, const int64_t* classes, int Ncls, cudaStream_t s);

}  // namespace ivid
