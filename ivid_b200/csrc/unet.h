// ADM UNet: topology / state-dict schema (host), packed device weights, per-batch execution plan.
// Mirrors the constructor logic of the reference's AdmUnet2d (diffusion/backbones/adm.py:318-487) so that the
// state-dict keys and shapes are identical (SURVEY.md §8b), but executes the forward (adm.py:526-566) as a static list
// of sm_90a kernel launches over NHWC tensors.
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/ivid_b200.h"
#include "ops.h"

namespace ivid {

struct UnetConfig {
  int image_size = 0, in_channels = 0, model_channels = 0, out_channels = 0, num_res_blocks = 0;
  std::vector<int> attention_resolutions;
  std::vector<double> channel_mult{1, 2, 4, 8};
  bool conv_resample = true;
  int num_classes = 0;            // 0 = not class conditional
  bool has_null_class = false;
  bool use_fp16 = false;
  int num_groups = 32;
  int num_heads = 1;
  int num_head_channels = -1;
  bool use_scale_shift_norm = true;
  bool resblock_updown = true;
  double dropout = 0.0;
};

struct ParamSpec {
  std::string name;
  std::vector<int64_t> shape;
  bool is_buffer = false;
  bool set = false;
  std::vector<float> host;
  size_t numel() const { size_t n = 1; for (auto d : shape) n *= static_cast<size_t>(d); return n; }
};

// A conv's operands in the weight arena, as conv_pack lays them out: fp16 columns [cout_pad][K] at w_off (none when K == 0)
// and the bias at b_off.  fp8: segment 0 runs as e4m3 from its columns at w8_off, and the fp16 columns are only the skip
// segments', all scaled by 2^e8.  Unet::build_plan binds them to a ConvDesc.
struct ConvW { int cout = 0, cout_pad = 0, K = 0; size_t w_off = 0, b_off = 0; bool fp8 = false; int e8 = 0; size_t w8_off = 0; };
struct GnW { int C = 0; size_t g_off = 0, b_off = 0; };
struct LinW { int O = 0, K = 0; size_t w_off = 0, b_off = 0; };

struct ResBlockDef {
  std::string pfx;
  int cin = 0, cout = 0;
  int cat0 = 0;            // up-path ResBlocks: width of the first part (h) of the concatenated input [h, skip]; 0 otherwise
  int mode = 0;            // 0 same, 1 up, 2 down
  bool skip_conv = false;
  int film_off = 0;        // column offset of this block's (scale|shift) in the FiLM table
  GnW gn1, gn2;
  ConvW conv1, conv2;      // conv2 holds out_layers.3 (+ skip_connection as extra K columns, one K segment per concat part)
};
struct AttnBlockDef {
  std::string pfx;
  int C = 0;
  int head_ch = 64;        // channels per head (a multiple of 64)
  GnW gn;
  ConvW qkv, proj;
};
struct ResampleDef {       // plain Downsample2d / Upsample2d layer (resblock_updown=False, adm.py:60-117)
  std::string pfx;         // layer name ("input_blocks.3.0", "output_blocks.2.1")
  int C = 0;
  int mode = 0;            // 1 up (nearest 2x [+ conv 3x3]), 2 down (conv 3x3 stride 2, or AvgPool2d(2))
  bool conv = false;       // conv_resample
  ConvW w;                 // op / conv weights, packed as an ordinary 3x3 conv
};
enum class LayerKind { kResBlock, kAttention, kResample };   // kResample: plain Downsample2d / Upsample2d layer
struct LayerRef { LayerKind kind; int idx; };                 // idx into res_, attn_ or resample_
struct BlockDef { std::vector<LayerRef> layers; bool is_input = false; bool is_output = false; };

struct Plan;

// Optional replacement of the output head's last kernel (eps_gather_kernel): the sampler hands the forward a launcher that
// consumes the tap columns Y directly (step_kernel<HeadTaps, ...>: eps of both guidance halves -> mix -> x_{t-1}), so that eps never
// goes to HBM and the update is the last node of the forward's CUDA graph.  `key` must change whenever anything the launcher
// bakes in (pointers, scalars) changes: it is part of the graph-cache key.
struct HeadHook {
  std::function<void(const float* Y, const float* bias, int N, int H, int W, int Co, int ldy, cudaStream_t s)> launch;
  uint64_t key = 0;
};

// Perturbed-attention guidance (PAG, Ahn et al. 2024, arXiv:2403.17377): rows [row0, N) of a forward replace the attention
// map of every listed attention layer (indices into the attention layers in state-dict order) by the identity, so those
// layers output their V channels.  Rows [0, row0) run the ordinary forward.  No layers (or row0 = N): no perturbation.
struct AttnPerturb {
  int row0 = 0;
  std::vector<int> layers;
};

class Unet {
 public:
  explicit Unet(const std::string& cfg_json);
  ~Unet();

  const UnetConfig& cfg() const { return cfg_; }
  const std::vector<ParamSpec>& params() const { return params_; }
  void set_param(const std::string& name, const float* data, const int64_t* shape, int ndim);
  void finalize(int device);
  // 0 = fp16 operands everywhere (default), 1 = e4m3 operands for the ResBlock 3x3 convs (DESIGN.md §2); takes effect at
  // the next finalize
  void set_precision(int precision);
  bool finalized() const { return arena_ != nullptr; }
  void* arena() const { return arena_; }
  size_t arena_bytes() const { return arena_bytes_; }
  int device() const { return device_; }

  // forward over a batch of N samples of H x W pixels; x rows are read modulo Nx (CFG halves share x).
  // cache_branch = -1: the full forward.  0 <= cache_branch <= num_res_blocks: the reuse forward at that branch (DeepCache,
  // include/ivid_b200.h), which runs the embeddings, input packing, input blocks 0..b, output blocks L-1-b..L-1 and the head,
  // and reads the output of output block L-2-b that the plan's last full forward left in place; kErrState before any full
  // forward of the plan.
  // pert: perturbed rows and layers (nullptr: none).  A perturbed forward runs on a plan of its own, keyed by the
  // perturbation as well as (N, H, W), so its graphs and its feature cache are never shared with an unperturbed forward.
  void forward(const float* x, int Nx, int H, int W, const ivid_cond_t* cond, const int64_t* t, const int64_t* classes,
               float* eps, int N, cudaStream_t stream, const HeadHook* hook = nullptr, int cache_branch = -1,
               const AttnPerturb* pert = nullptr);
  // attention layers in state-dict order: their count and names ("middle_block.1", "input_blocks.7.1", ...)
  int num_attention_layers() const { return static_cast<int>(attn_.size()); }
  const std::string& attention_layer_name(int i) const { return attn_.at(i).pfx; }
  // whether the output head of an H x W forward runs as the tap-column GEMM whose last kernel a HeadHook can replace
  bool can_fuse_head(int W) const;
  // inputs the network accepts: H and W positive multiples of 2^(levels - 1), as in the reference (its skip concatenations
  // fail otherwise); kErrState otherwise
  void check_geometry(int H, int W) const;
  // Device-resident Philox stream id (step counter) of the conditional-input noise: the sampler points this at its step
  // state so that consecutive denoising steps replay the same CUDA graph (a by-value stream id would change the key).
  void set_cond_stream_dev(const int* p) { cond_stream_dev_ = p; }
  void debug_tap(int N, const std::string& name, float* host_out, size_t capacity, int* C, int* H, int* W);
  // per-kernel-family timing of the forwards issued between begin/end (CUDA events around every launch)
  void profile_begin();
  std::string profile_end();    // JSON: {"label": {"launches", "ms", "flops", "bytes"}, ...}

 private:
  void build_topology();
  int add_param(const std::string& name, std::vector<int64_t> shape, bool is_buffer = false);
  const ParamSpec& P(const std::string& name) const;
  Plan* get_plan(int N, int H, int W, const AttnPerturb& pert);
  Plan* build_plan(int N, int H, int W, const AttnPerturb& pert);

  UnetConfig cfg_;
  int embed_dim_ = 0;
  std::vector<ParamSpec> params_;
  std::map<std::string, int> pindex_;
  std::vector<ResBlockDef> res_;
  std::vector<AttnBlockDef> attn_;
  std::vector<ResampleDef> resample_;
  std::vector<BlockDef> blocks_;     // input blocks (block 0 = input conv, no layers), middle, output blocks in order
  int film_total_ = 0;
  int in_ch_stem_ = 0;               // channels after the input conv
  int final_ch_ = 0;
  int precision_ = 0;

  // packed weights
  ConvW in_conv_, out_conv_;
  ConvW out1x1_;                     // split-precision 1x1 form of the output conv (9*Co tap columns), see unet.cu
  bool out_split_ = false;
  GnW out_gn_;
  LinW te1_, te2_, film_;
  size_t freqs_off_ = 0, label_off_ = 0;
  uint8_t* arena_ = nullptr;
  size_t arena_bytes_ = 0;
  int device_ = -1;

  const int* cond_stream_dev_ = nullptr;
  cudaStream_t cap_stream_ = nullptr;
  struct ProfAgg { int launches = 0; double ms = 0, flops = 0, bytes = 0; };
  bool profile_ = false;
  std::map<std::string, ProfAgg> profile_acc_;
  std::string profile_ops_;
  std::vector<std::unique_ptr<Plan>> plans_;       // keyed by (N, H, W, perturbation)
  uint64_t plan_uses_ = 0;                         // debug_tap reads the most recently run plan of a batch size
  friend struct Plan;
};

}  // namespace ivid
