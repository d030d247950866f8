// C ABI (include/ivid_b200.h): exception -> status-code translation, op-level entry points.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/ivid_b200.h"
#include "ops.h"
#include "sampler.h"
#include "unet.h"

using namespace ivid;

struct ivid_unet { std::unique_ptr<Unet> impl; };
struct ivid_sampler { std::unique_ptr<Sampler> impl; };

static thread_local std::string g_last_error;
namespace ivid { void set_last_error(const std::string& msg) { g_last_error = msg; } }

template <class F>
static int guarded(F&& f) {
  try {
    f();
    return IVID_OK;
  } catch (const Error& e) {
    g_last_error = e.what();
    return e.code;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return IVID_ERR_STATE;
  } catch (...) {
    g_last_error = "unknown error";
    return IVID_ERR_STATE;
  }
}

#define IVID_NOT_NULL(p) IVID_REQUIRE((p) != nullptr, #p " must not be NULL")

extern "C" {

const char* ivid_last_error(void) { return g_last_error.c_str(); }
int ivid_version(void) { return 100; }

int ivid_device_info(int device, int* sm_count_out, int* cc_major, int* cc_minor) {
  return guarded([&] {
    cudaDeviceProp prop;
    IVID_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
    if (sm_count_out) *sm_count_out = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
  });
}

int ivid_unet_create(const char* cfg_json, ivid_unet_t** out) {
  return guarded([&] {
    IVID_NOT_NULL(cfg_json);
    IVID_NOT_NULL(out);
    auto h = std::make_unique<ivid_unet>();
    h->impl = std::make_unique<Unet>(std::string(cfg_json));
    *out = h.release();
  });
}
int ivid_unet_destroy(ivid_unet_t* h) {
  return guarded([&] { delete h; });
}
int ivid_unet_num_params(const ivid_unet_t* h, int* count) {
  return guarded([&] {
    IVID_NOT_NULL(h); IVID_NOT_NULL(count);
    *count = static_cast<int>(h->impl->params().size());
  });
}
int ivid_unet_param_info(const ivid_unet_t* h, int index, const char** name, int64_t shape[4], int* ndim, int* is_buffer) {
  return guarded([&] {
    IVID_NOT_NULL(h);
    const auto& ps = h->impl->params();
    IVID_REQUIRE(index >= 0 && index < static_cast<int>(ps.size()), "parameter index out of range");
    const ParamSpec& p = ps[index];
    if (name) *name = p.name.c_str();
    if (ndim) *ndim = static_cast<int>(p.shape.size());
    if (shape) for (size_t i = 0; i < 4; ++i) shape[i] = i < p.shape.size() ? p.shape[i] : 1;
    if (is_buffer) *is_buffer = p.is_buffer ? 1 : 0;
  });
}
int ivid_unet_set_param(ivid_unet_t* h, const char* name, const float* host_data, const int64_t* shape, int ndim) {
  return guarded([&] {
    IVID_NOT_NULL(h); IVID_NOT_NULL(name); IVID_NOT_NULL(host_data); IVID_NOT_NULL(shape);
    h->impl->set_param(name, host_data, shape, ndim);
  });
}
int ivid_unet_finalize(ivid_unet_t* h, int device) {
  return guarded([&] {
    IVID_NOT_NULL(h);
    h->impl->finalize(device);
  });
}
int ivid_unet_set_precision(ivid_unet_t* h, int precision) {
  return guarded([&] {
    IVID_NOT_NULL(h);
    h->impl->set_precision(precision);
  });
}
int ivid_fp8_e4m3_quantize(const float* in, uint8_t* out, uint64_t count) {
  return guarded([&] {
    IVID_REQUIRE(count == 0 || (in != nullptr && out != nullptr), "in and out must not be NULL");
    for (uint64_t i = 0; i < count; ++i) out[i] = fp8_e4m3_from_float(in[i]);
  });
}
int ivid_fp8_weight_exponent(const float* w, uint64_t count, int* e_out) {
  return guarded([&] {
    IVID_REQUIRE(count == 0 || w != nullptr, "w must not be NULL");
    IVID_NOT_NULL(e_out);
    float mx = 0.f;
    for (uint64_t i = 0; i < count; ++i) mx = std::max(mx, std::fabs(w[i]));
    *e_out = fp8_weight_exponent(mx);
  });
}
int ivid_unet_weight_arena(const ivid_unet_t* h, void** dev_ptr, uint64_t* bytes) {
  return guarded([&] {
    IVID_NOT_NULL(h);
    if (!h->impl->finalized()) throw Error(kErrState, "weight arena requested before finalize");
    if (dev_ptr) *dev_ptr = h->impl->arena();
    if (bytes) *bytes = h->impl->arena_bytes();
  });
}
int ivid_unet_forward_hw(ivid_unet_t* h, const float* x_dev, int Nx, int H, int W, const ivid_cond_t* cond,
                         const int64_t* t_dev, const int64_t* classes_dev, float* eps_dev, int N, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(h); IVID_NOT_NULL(x_dev); IVID_NOT_NULL(t_dev); IVID_NOT_NULL(eps_dev);
    h->impl->forward(x_dev, Nx, H, W, cond, t_dev, classes_dev, eps_dev, N, static_cast<cudaStream_t>(stream));
  });
}
int ivid_unet_forward_reuse(ivid_unet_t* h, const float* x_dev, int Nx, int H, int W, const ivid_cond_t* cond,
                            const int64_t* t_dev, const int64_t* classes_dev, float* eps_dev, int N, int cache_branch,
                            void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(h); IVID_NOT_NULL(x_dev); IVID_NOT_NULL(t_dev); IVID_NOT_NULL(eps_dev);
    IVID_REQUIRE(cache_branch >= 0, "cache_branch must be in [0, num_res_blocks]");
    h->impl->forward(x_dev, Nx, H, W, cond, t_dev, classes_dev, eps_dev, N, static_cast<cudaStream_t>(stream), nullptr,
                     cache_branch);
  });
}
int ivid_unet_forward_perturbed(ivid_unet_t* h, const float* x_dev, int Nx, int H, int W, const ivid_cond_t* cond,
                                const int64_t* t_dev, const int64_t* classes_dev, float* eps_dev, int N, int row0,
                                const int* layers_host, int num_layers, int cache_branch, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(h); IVID_NOT_NULL(x_dev); IVID_NOT_NULL(t_dev); IVID_NOT_NULL(eps_dev);
    IVID_REQUIRE(num_layers >= 1 && layers_host != nullptr, "perturbed forward: at least one attention layer");
    IVID_REQUIRE(row0 >= 0 && row0 <= N, "perturbed forward: row0 must lie in [0, N]");
    AttnPerturb pert;
    pert.row0 = row0;
    pert.layers.assign(layers_host, layers_host + num_layers);
    h->impl->forward(x_dev, Nx, H, W, cond, t_dev, classes_dev, eps_dev, N, static_cast<cudaStream_t>(stream), nullptr,
                     cache_branch, &pert);
  });
}
// the square forwards at the backbone's image_size
int ivid_unet_forward(ivid_unet_t* h, const float* x_dev, int Nx, const int64_t* t_dev, const int64_t* classes_dev,
                      float* eps_dev, int N, void* stream) {
  const int S = h != nullptr ? h->impl->cfg().image_size : 0;
  return ivid_unet_forward_hw(h, x_dev, Nx, S, S, nullptr, t_dev, classes_dev, eps_dev, N, stream);
}
int ivid_unet_forward_cond(ivid_unet_t* h, const float* x_dev, int Nx, const ivid_cond_t* cond, const int64_t* t_dev,
                           const int64_t* classes_dev, float* eps_dev, int N, void* stream) {
  if (cond == nullptr) return guarded([&] { IVID_NOT_NULL(cond); });
  const int S = h != nullptr ? h->impl->cfg().image_size : 0;
  return ivid_unet_forward_hw(h, x_dev, Nx, S, S, cond, t_dev, classes_dev, eps_dev, N, stream);
}

int ivid_conv_tile(int H, int W, int* tw, int* th, int* tn, int* fused_stats) {
  return guarded([&] {
    int a, b, c;
    conv_tile(H, W, &a, &b, &c);
    if (tw) *tw = a;
    if (th) *th = b;
    if (tn) *tn = c;
    if (fused_stats) *fused_stats = conv_can_fuse_stats(H, W) ? 1 : 0;
  });
}

int ivid_unet_debug_tap(ivid_unet_t* h, int N, const char* layer, float* host_out, uint64_t capacity, int* C, int* H, int* W) {
  return guarded([&] {
    IVID_NOT_NULL(h); IVID_NOT_NULL(layer);
    h->impl->debug_tap(N, layer, host_out, static_cast<size_t>(capacity), C, H, W);
  });
}

int ivid_unet_profile_begin(ivid_unet_t* h) {
  return guarded([&] { IVID_NOT_NULL(h); h->impl->profile_begin(); });
}
int ivid_unet_profile_end(ivid_unet_t* h, char* json_out, int capacity) {
  return guarded([&] {
    IVID_NOT_NULL(h); IVID_NOT_NULL(json_out);
    const std::string js = h->impl->profile_end();
    IVID_REQUIRE(static_cast<int>(js.size()) < capacity, "profile buffer too small");
    std::memcpy(json_out, js.c_str(), js.size() + 1);
  });
}

int ivid_sampler_create(const double* betas, int timesteps, ivid_sampler_t** out) {
  return guarded([&] {
    IVID_NOT_NULL(betas); IVID_NOT_NULL(out);
    auto s = std::make_unique<ivid_sampler>();
    s->impl = std::make_unique<Sampler>(betas, timesteps);
    *out = s.release();
  });
}
int ivid_sampler_destroy(ivid_sampler_t* s) {
  return guarded([&] { delete s; });
}
int ivid_sampler_table(const ivid_sampler_t* s, int which, double* out, int count) {
  return guarded([&] {
    IVID_NOT_NULL(s); IVID_NOT_NULL(out);
    const auto& t = s->impl->table(which);
    IVID_REQUIRE(count == static_cast<int>(t.size()), "table length mismatch");
    std::memcpy(out, t.data(), sizeof(double) * t.size());
  });
}
int ivid_sampler_step(ivid_sampler_t* s, ivid_unet_t* unet, const float* x_t_dev, float* x_prev_dev, float* pred_x0_dev,
                      int N, int t, int t_prev, const ivid_step_args_t* args, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(s); IVID_NOT_NULL(unet); IVID_NOT_NULL(x_t_dev); IVID_NOT_NULL(x_prev_dev); IVID_NOT_NULL(args);
    s->impl->step(*unet->impl, x_t_dev, x_prev_dev, pred_x0_dev, N, t, t_prev, *args, t, static_cast<cudaStream_t>(stream));
  });
}
int ivid_sampler_step_dev(ivid_sampler_t* s, ivid_unet_t* unet, const float* x_t_dev, float* x_prev_dev, float* pred_x0_dev,
                          int N, const int64_t* t_dev, const int64_t* t_prev_dev, const ivid_step_args_t* args, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(s); IVID_NOT_NULL(unet); IVID_NOT_NULL(x_t_dev); IVID_NOT_NULL(x_prev_dev); IVID_NOT_NULL(args); IVID_NOT_NULL(t_dev);
    IVID_REQUIRE(args->kind == 0 || t_prev_dev != nullptr, "DDIM / DPM-Solver++ step needs t_prev");
    s->impl->step(*unet->impl, x_t_dev, x_prev_dev, pred_x0_dev, N, 0, 0, *args, 0, static_cast<cudaStream_t>(stream), t_dev, t_prev_dev);
  });
}
int ivid_cfg_mix(const float* eps2n_dev, float strength, float* out_dev, uint64_t count, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(eps2n_dev); IVID_NOT_NULL(out_dev);
    launch_cfg_mix(eps2n_dev, out_dev, static_cast<size_t>(count), strength, static_cast<cudaStream_t>(stream));
  });
}
int ivid_guidance_mix(const float* eps_dev, uint64_t count, int cfg, float strength, int pag, float pag_scale, float* out_dev,
                      void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(eps_dev); IVID_NOT_NULL(out_dev);
    launch_guidance_mix(eps_dev, out_dev, static_cast<size_t>(count), cfg, strength, pag, pag_scale, static_cast<cudaStream_t>(stream));
  });
}
int ivid_op_dynamic_threshold(const float* x_dev, int N, int M, double ratio, double threshold_max, float* s_out_dev,
                              float* x_out_dev, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(x_dev); IVID_NOT_NULL(s_out_dev); IVID_NOT_NULL(x_out_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    launch_dynamic_threshold(x_dev, N, M, ratio, threshold_max, s_out_dev, x_out_dev, st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  });
}
int ivid_op_apg(const float* d_c_dev, const float* d_u_dev, float* state_inout_dev, int N, int M, float s, double eta,
                double r, double beta, float* out_dev, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(d_c_dev); IVID_NOT_NULL(d_u_dev); IVID_NOT_NULL(state_inout_dev); IVID_NOT_NULL(out_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    launch_apg(d_c_dev, d_u_dev, state_inout_dev, N, M, s, eta, r, beta, out_dev, st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  });
}
int ivid_sampler_run(ivid_sampler_t* s, ivid_unet_t* unet, float* x_inout_dev, int N, int steps,
                     const ivid_step_args_t* args, const float* noise_all_dev, const float* cond_noise_all_dev,
                     float* traj_x0_dev, float* traj_xt_dev, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(s); IVID_NOT_NULL(unet); IVID_NOT_NULL(x_inout_dev); IVID_NOT_NULL(args);
    s->impl->run(*unet->impl, x_inout_dev, N, steps, *args, noise_all_dev, cond_noise_all_dev, traj_x0_dev, traj_xt_dev,
                 static_cast<cudaStream_t>(stream));
  });
}
int ivid_sampler_diffuse(ivid_sampler_t* s, const float* x0_dev, const float* noise_dev, int N, uint64_t count_per_sample,
                         int t, uint64_t seed, float* out_dev, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(s); IVID_NOT_NULL(x0_dev); IVID_NOT_NULL(out_dev);
    s->impl->diffuse(x0_dev, noise_dev, N, static_cast<size_t>(count_per_sample), t, seed, out_dev,
                     static_cast<cudaStream_t>(stream));
  });
}

// ------------------------------------------------------------------------------------------------------------------
// operator-level entry points (weights are packed per call: test / profiling paths, not the hot loop)
// ------------------------------------------------------------------------------------------------------------------
namespace {
struct DevBuf {
  void* p = nullptr;                                 // stays null for zero bytes
  explicit DevBuf(size_t bytes) { if (bytes > 0) IVID_CHECK_CUDA(cudaMalloc(&p, bytes)); }
  ~DevBuf() { if (p) cudaFree(p); }
  DevBuf(const DevBuf&) = delete;
};
}  // namespace

// One conv as the network builds it: packed by conv_pack (cin2a = C1 for a skip over two tensors), every ConvDesc field the
// network sets taken from the arguments, and conv_launch_create left to reject the combinations it does not run.
int ivid_op_conv2d_ex(const ivid_op_conv_t* a, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(a);
    IVID_NOT_NULL(a->act0_dev); IVID_NOT_NULL(a->w0_host); IVID_NOT_NULL(a->out_dev);
    IVID_REQUIRE(a->ksize == 3 || a->ksize == 1, "conv: kernel size must be 3 or 1");
    IVID_REQUIRE(a->C0 > 0 && a->C0 % 8 == 0 && a->C1 % 8 == 0 && a->C2 % 8 == 0, "conv: channels must be multiples of 8");
    IVID_REQUIRE(a->act1_dev == nullptr || a->wskip_host != nullptr, "conv: a skip input needs its weights (w2_host; wskip_host of ivid_op_conv2d_ex)");
    IVID_REQUIRE(a->act2_dev == nullptr || (a->act1_dev != nullptr && a->C2 > 0), "conv: act2_dev is the second part of a skip over act1_dev");
    IVID_REQUIRE(a->out_mode >= 0 && a->out_mode <= 2, "conv: out_mode must be 0, 1 or 2");
    const int C1 = a->act1_dev ? a->C1 : 0, C2 = a->act2_dev ? a->C2 : 0;
    const ConvPack pk = conv_pack(a->w0_host, a->b0_host, a->Cout, a->C0, a->ksize, conv_pad_k(a->C0), C1 ? a->wskip_host : nullptr,
                                  C1 ? a->bskip_host : nullptr, C1 + C2, C2 ? C1 : 0, a->e4m3 != 0);
    if (pk.refused != nullptr) throw Error(kErrInvalidArgument, std::string("conv: no e4m3 form: ") + pk.refused);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevBuf dw8(pk.w8.size()), dw(pk.w16.size() * 2), db(pk.bias.size() * 4);
    if (pk.e4m3) IVID_CHECK_CUDA(cudaMemcpyAsync(dw8.p, pk.w8.data(), pk.w8.size(), cudaMemcpyHostToDevice, st));
    if (pk.K > 0) IVID_CHECK_CUDA(cudaMemcpyAsync(dw.p, pk.w16.data(), pk.w16.size() * 2, cudaMemcpyHostToDevice, st));
    IVID_CHECK_CUDA(cudaMemcpyAsync(db.p, pk.bias.data(), pk.bias.size() * 4, cudaMemcpyHostToDevice, st));
    ConvDesc d;
    d.act0 = a->act0_dev; d.C0 = a->C0; d.taps0 = a->ksize * a->ksize;
    if (C1) { d.act1 = a->act1_dev; d.C1 = C1; d.taps1 = 1; }
    if (C2) { d.act2 = a->act2_dev; d.C2 = C2; d.taps2 = 1; }
    d.weight = dw.p; d.weight8 = dw8.p; d.acc_scale = std::ldexp(1.0f, -pk.e);
    d.cout_pad = pk.cout_pad; d.cout = a->Cout; d.bias = static_cast<const float*>(db.p);
    d.residual = a->residual_dev; d.ldr = a->Cout; d.residual_up = a->residual_up != 0;
    d.out = a->out_dev; d.ldc = a->Cout; d.out_mode = a->out_mode; d.out16 = a->out16_dev; d.stats = a->stats_dev;
    d.N = a->N; d.H = a->H; d.W = a->W;
    std::unique_ptr<ConvLaunch, void (*)(ConvLaunch*)> l(conv_launch_create(d), conv_launch_destroy);
    conv_launch_run(l.get(), st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
    if (a->e_out) *a->e_out = pk.e;
  });
}

static int op_conv2d(const void* act_dev, int N, int H, int W, int Cin, const float* w_host, const float* bias_host, int Cout,
                     int ksize, const void* act2_dev, int Cin2, const float* w2_host, const float* bias2_host,
                     const float* residual_dev, void* out_dev, int out_fp16, bool e4m3, int* e_out, void* stream) {
  ivid_op_conv_t a{};
  a.act0_dev = act_dev; a.C0 = Cin; a.ksize = ksize; a.w0_host = w_host; a.b0_host = bias_host;
  a.e4m3 = e4m3 ? 1 : 0; a.e_out = e_out;
  a.act1_dev = act2_dev; a.C1 = act2_dev ? Cin2 : 0; a.wskip_host = w2_host; a.bskip_host = bias2_host;
  a.residual_dev = residual_dev;
  a.N = N; a.H = H; a.W = W; a.Cout = Cout;
  a.out_dev = out_dev; a.out_mode = out_fp16 ? 1 : 0;
  return ivid_op_conv2d_ex(&a, stream);
}

int ivid_op_conv2d(const void* act_dev, int N, int H, int W, int Cin, const float* w_host, const float* bias_host,
                   int Cout, int ksize, const void* act2_dev, int Cin2, const float* w2_host, const float* bias2_host,
                   const float* residual_dev, void* out_dev, int out_fp16, void* stream) {
  return op_conv2d(act_dev, N, H, W, Cin, w_host, bias_host, Cout, ksize, act2_dev, Cin2, w2_host, bias2_host, residual_dev,
                   out_dev, out_fp16, false, nullptr, stream);
}
int ivid_op_conv2d_e4m3(const void* act_dev, int N, int H, int W, int Cin, const float* w_host, const float* bias_host,
                        int Cout, int ksize, const void* act2_dev, int Cin2, const float* w2_host, const float* bias2_host,
                        const float* residual_dev, void* out_dev, int out_fp16, int* e_out, void* stream) {
  return op_conv2d(act_dev, N, H, W, Cin, w_host, bias_host, Cout, ksize, act2_dev, Cin2, w2_host, bias2_host, residual_dev,
                   out_dev, out_fp16, true, e_out, stream);
}

// One GroupNorm apply as the network launches it; statistics a caller does not supply are taken here by gn_stats (fp32
// sources).  launch_gn_apply rejects the combinations the network does not run.
int ivid_op_group_norm_apply(const ivid_op_gn_t* a, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(a);
    IVID_NOT_NULL(a->x0_dev); IVID_NOT_NULL(a->gamma_host); IVID_NOT_NULL(a->beta_host); IVID_NOT_NULL(a->out_dev);
    const int N = a->N, HW = a->H * a->W, C0 = a->C0, C1 = a->x1_dev ? a->C1 : 0, C = C0 + C1;
    IVID_REQUIRE(N > 0 && HW > 0 && C0 > 0, "group norm: empty tensor");
    IVID_REQUIRE(a->film_dev == nullptr || a->film_ld >= a->film_off + (a->film_add ? C : 2 * C),
                 "group norm: the FiLM row (film_off + C, or + 2C with a shift) must fit film_ld");
    const bool need0 = a->stats0_dev == nullptr, need1 = C1 > 0 && a->stats1_dev == nullptr;
    IVID_REQUIRE(!(need0 || need1) || !a->x_fp16, "group norm: statistics of fp16 sources must be supplied");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevBuf dg(C * 4), dbt(C * 4), st0(need0 ? static_cast<size_t>(N) * C0 * 16 : 0), st1(need1 ? static_cast<size_t>(N) * C1 * 16 : 0);
    IVID_CHECK_CUDA(cudaMemcpyAsync(dg.p, a->gamma_host, C * 4, cudaMemcpyHostToDevice, st));
    IVID_CHECK_CUDA(cudaMemcpyAsync(dbt.p, a->beta_host, C * 4, cudaMemcpyHostToDevice, st));
    if (need0) {
      IVID_CHECK_CUDA(cudaMemsetAsync(st0.p, 0, static_cast<size_t>(N) * C0 * 16, st));
      launch_gn_stats(static_cast<const float*>(a->x0_dev), static_cast<double*>(st0.p), N, HW, C0, st);
    }
    if (need1) {
      IVID_CHECK_CUDA(cudaMemsetAsync(st1.p, 0, static_cast<size_t>(N) * C1 * 16, st));
      launch_gn_stats(static_cast<const float*>(a->x1_dev), static_cast<double*>(st1.p), N, HW, C1, st);
    }
    GnApplyDesc g;
    g.x0 = a->x0_dev; g.x1 = C1 > 0 ? a->x1_dev : nullptr; g.C0 = C0; g.C1 = C1; g.x0_half = a->x_fp16 != 0;
    g.N = N; g.H = a->H; g.W = a->W; g.mode = a->mode; g.silu = a->silu;
    g.stats0 = need0 ? static_cast<const double*>(st0.p) : a->stats0_dev;
    g.stats1 = C1 == 0 ? nullptr : (need1 ? static_cast<const double*>(st1.p) : a->stats1_dev);
    g.groups = a->groups; g.eps = a->eps; g.gamma = static_cast<float*>(dg.p); g.beta = static_cast<float*>(dbt.p);
    g.film = a->film_dev; g.film_ld = a->film_ld; g.film_off = a->film_off; g.film_add = a->film_add != 0;
    g.out_act = a->out_dev; g.out_e4m3 = a->out_e4m3 != 0; g.out_lo = a->out_lo_dev;
    g.out_raw16 = a->out_raw16_dev; g.out_raw32 = a->out_raw32_dev;
    launch_gn_apply(g, st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  });
}

int ivid_op_gn_stats(const float* x_dev, int N, int H, int W, int C, double* stats_dev, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(x_dev); IVID_NOT_NULL(stats_dev);
    IVID_REQUIRE(N > 0 && N <= 65535 && H > 0 && W > 0 && C > 0 && C % 4 == 0,
                 "gn_stats: N in [1, 65535], positive H and W, C a positive multiple of 4");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    launch_gn_stats(x_dev, stats_dev, N, H * W, C, st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  });
}

// One Downsample2d / Upsample2d with the launches and descriptor fields of run_resample in unet.cu: the same weight pitch
// (C for the stride-2 conv's gathered taps, conv_pad_k(C) for the upsample conv), and the statistics from the conv
// epilogue where add_conv fuses them, from gn_stats otherwise and after every pooling / nearest layer.
int ivid_op_resample(const ivid_op_resample_t* a, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(a);
    IVID_NOT_NULL(a->x_dev); IVID_NOT_NULL(a->out_dev);
    IVID_REQUIRE(a->mode == 1 || a->mode == 2, "resample: mode must be 1 (up) or 2 (down)");
    IVID_REQUIRE(a->conv == 0 || a->conv == 1, "resample: conv must be 0 or 1");
    const int N = a->N, H = a->H, W = a->W, C = a->C;
    IVID_REQUIRE(N > 0 && N <= 65535 && H > 0 && W > 0 && C > 0 && C % 8 == 0,
                 "resample: N in [1, 65535], positive H and W, C a positive multiple of 8");
    IVID_REQUIRE(a->mode == 1 || (H % 2 == 0 && W % 2 == 0), "resample: downsampling needs an even H and W");
    IVID_REQUIRE(a->conv == 1 || a->operand_dev == nullptr, "resample: operand_dev belongs to the conv forms");
    if (a->conv) IVID_NOT_NULL(a->w_host);
    const int Ho = a->mode == 1 ? 2 * H : H / 2, Wo = a->mode == 1 ? 2 * W : W / 2;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (a->conv) {
      const ConvPack pk = conv_pack(a->w_host, a->b_host, C, C, 3, a->mode == 2 ? C : conv_pad_k(C), nullptr, nullptr, 0, 0, false);
      const size_t op_elems = static_cast<size_t>(N) * Ho * Wo * (a->mode == 2 ? 9 * C : C);
      DevBuf dw(pk.w16.size() * 2), db(pk.bias.size() * 4), dop(a->operand_dev ? 0 : op_elems * 2);
      void* opnd = a->operand_dev ? a->operand_dev : dop.p;
      IVID_CHECK_CUDA(cudaMemcpyAsync(dw.p, pk.w16.data(), pk.w16.size() * 2, cudaMemcpyHostToDevice, st));
      IVID_CHECK_CUDA(cudaMemcpyAsync(db.p, pk.bias.data(), pk.bias.size() * 4, cudaMemcpyHostToDevice, st));
      ConvDesc d;
      d.act0 = opnd; d.C0 = a->mode == 2 ? 9 * C : C; d.taps0 = a->mode == 2 ? 1 : 9;
      d.weight = dw.p; d.cout_pad = pk.cout_pad; d.cout = C; d.bias = static_cast<const float*>(db.p);
      d.out = a->out_dev; d.out16 = a->out16_dev; d.out_mode = 0; d.ldc = C; d.N = N; d.H = Ho; d.W = Wo;
      const bool fused = a->stats_dev != nullptr && conv_can_fuse_stats(Ho, Wo);
      if (fused) d.stats = a->stats_dev;
      std::unique_ptr<ConvLaunch, void (*)(ConvLaunch*)> l(conv_launch_create(d), conv_launch_destroy);   // may refuse: before any launch
      if (a->mode == 2) launch_im2col_s2(a->x_dev, opnd, N, H, W, C, st);
      else launch_upsample2x_h16(a->x_dev, opnd, N, H, W, C, st);
      conv_launch_run(l.get(), st);
      if (a->stats_dev != nullptr && !fused) launch_gn_stats(a->out_dev, a->stats_dev, N, Ho * Wo, C, st);
    } else {
      launch_resample_f32(static_cast<const float*>(a->x_dev), a->out_dev, a->out16_dev, N, H, W, C, a->mode, st);
      if (a->stats_dev != nullptr) launch_gn_stats(a->out_dev, a->stats_dev, N, Ho * Wo, C, st);
    }
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  });
}

static int op_group_norm(const float* x0_dev, int C0, const float* x1_dev, int C1, int N, int H, int W, int groups,
                         float eps, const float* gamma_host, const float* beta_host, const float* film_dev, int silu,
                         int mode, void* out_dev, bool e4m3, void* stream) {
  ivid_op_gn_t a{};
  a.x0_dev = x0_dev; a.C0 = C0; a.x1_dev = x1_dev; a.C1 = x1_dev ? C1 : 0;
  a.N = N; a.H = H; a.W = W; a.groups = groups; a.eps = eps; a.gamma_host = gamma_host; a.beta_host = beta_host;
  a.film_dev = film_dev; a.film_ld = 2 * (a.C0 + a.C1); a.film_off = 0;
  a.silu = silu; a.mode = mode; a.out_dev = out_dev; a.out_e4m3 = e4m3 ? 1 : 0;
  return ivid_op_group_norm_apply(&a, stream);
}

int ivid_op_group_norm(const float* x0_dev, int C0, const float* x1_dev, int C1, int N, int H, int W, int groups,
                       float eps, const float* gamma_host, const float* beta_host, const float* film_dev, int silu,
                       int mode, void* out_fp16_dev, void* stream) {
  return op_group_norm(x0_dev, C0, x1_dev, C1, N, H, W, groups, eps, gamma_host, beta_host, film_dev, silu, mode, out_fp16_dev,
                       false, stream);
}
int ivid_op_group_norm_e4m3(const float* x0_dev, int C0, const float* x1_dev, int C1, int N, int H, int W, int groups,
                            float eps, const float* gamma_host, const float* beta_host, const float* film_dev, int silu,
                            int mode, void* out_e4m3_dev, void* stream) {
  return op_group_norm(x0_dev, C0, x1_dev, C1, N, H, W, groups, eps, gamma_host, beta_host, film_dev, silu, mode, out_e4m3_dev,
                       true, stream);
}

int ivid_op_attention(const void* qkv_dev, int N, int T, int C, void* out_dev, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(qkv_dev); IVID_NOT_NULL(out_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::unique_ptr<AttnLaunch, void (*)(AttnLaunch*)> l(attn_launch_create(qkv_dev, N, T, C, 64, out_dev), attn_launch_destroy);
    attn_launch_run(l.get(), st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  });
}

int ivid_op_attention_heads(const void* qkv_dev, int N, int T, int C, int head_channels, void* out_dev, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(qkv_dev); IVID_NOT_NULL(out_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::unique_ptr<AttnLaunch, void (*)(AttnLaunch*)> l(attn_launch_create(qkv_dev, N, T, C, head_channels, out_dev), attn_launch_destroy);
    attn_launch_run(l.get(), st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  });
}

int ivid_op_attention_perturbed(const void* qkv_dev, int N, int T, int C, int head_channels, int row0, void* out_dev,
                                void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(qkv_dev); IVID_NOT_NULL(out_dev);
    IVID_REQUIRE(row0 >= 0 && row0 <= N, "attention: row0 must lie in [0, N]");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::unique_ptr<AttnLaunch, void (*)(AttnLaunch*)> l(attn_launch_create(qkv_dev, N, T, C, head_channels, out_dev, row0),
                                                         attn_launch_destroy);
    attn_launch_run(l.get(), st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  });
}

}  // extern "C"
