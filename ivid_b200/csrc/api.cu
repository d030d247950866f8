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
int ivid_sampler_run(ivid_sampler_t* s, ivid_unet_t* unet, float* x_inout_dev, int N, int steps,
                     const ivid_step_args_t* args, const float* noise_all_dev, const float* cond_noise_all_dev,
                     float* traj_x0_dev, float* traj_xt_dev, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(s); IVID_NOT_NULL(unet); IVID_NOT_NULL(x_inout_dev); IVID_NOT_NULL(args);
    s->impl->run(*unet->impl, x_inout_dev, N, steps, *args, noise_all_dev, cond_noise_all_dev, traj_x0_dev, traj_xt_dev,
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

// one conv, packed by conv_pack; e4m3: segment 0 in e4m3, and its weight exponent goes to e_out
static int op_conv2d(const void* act_dev, int N, int H, int W, int Cin, const float* w_host, const float* bias_host, int Cout,
                     int ksize, const void* act2_dev, int Cin2, const float* w2_host, const float* bias2_host,
                     const float* residual_dev, void* out_dev, int out_fp16, bool e4m3, int* e_out, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(act_dev); IVID_NOT_NULL(w_host); IVID_NOT_NULL(out_dev);
    IVID_REQUIRE(ksize == 3 || ksize == 1, "conv: kernel size must be 3 or 1");
    IVID_REQUIRE(Cin > 0 && Cin % 8 == 0 && Cin2 % 8 == 0, "conv: channels must be multiples of 8");
    IVID_REQUIRE(act2_dev == nullptr || w2_host != nullptr, "conv: a skip input (act2_dev) needs its weights (w2_host)");
    const ConvPack pk = conv_pack(w_host, bias_host, Cout, Cin, ksize, conv_pad_k(Cin), act2_dev ? w2_host : nullptr,
                                  act2_dev ? bias2_host : nullptr, act2_dev ? Cin2 : 0, 0, e4m3);
    if (pk.refused != nullptr) throw Error(kErrInvalidArgument, std::string("conv: no e4m3 form: ") + pk.refused);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    DevBuf dw8(pk.w8.size()), dw(pk.w16.size() * 2), db(pk.bias.size() * 4);
    if (pk.e4m3) IVID_CHECK_CUDA(cudaMemcpyAsync(dw8.p, pk.w8.data(), pk.w8.size(), cudaMemcpyHostToDevice, st));
    if (pk.K > 0) IVID_CHECK_CUDA(cudaMemcpyAsync(dw.p, pk.w16.data(), pk.w16.size() * 2, cudaMemcpyHostToDevice, st));
    IVID_CHECK_CUDA(cudaMemcpyAsync(db.p, pk.bias.data(), pk.bias.size() * 4, cudaMemcpyHostToDevice, st));
    ConvDesc d;
    d.act0 = act_dev; d.C0 = Cin; d.taps0 = ksize * ksize;
    if (act2_dev) { d.act1 = act2_dev; d.C1 = Cin2; d.taps1 = 1; }
    d.weight = dw.p; d.weight8 = dw8.p; d.acc_scale = std::ldexp(1.0f, -pk.e);
    d.cout_pad = pk.cout_pad; d.cout = Cout; d.bias = static_cast<const float*>(db.p);
    d.residual = residual_dev; d.ldr = Cout; d.out = out_dev; d.ldc = Cout; d.out_mode = out_fp16 ? 1 : 0;
    d.N = N; d.H = H; d.W = W;
    std::unique_ptr<ConvLaunch, void (*)(ConvLaunch*)> l(conv_launch_create(d), conv_launch_destroy);
    conv_launch_run(l.get(), st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
    if (e_out) *e_out = pk.e;
  });
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

static int op_group_norm(const float* x0_dev, int C0, const float* x1_dev, int C1, int N, int H, int W, int groups,
                         float eps, const float* gamma_host, const float* beta_host, const float* film_dev, int silu,
                         int mode, void* out_fp16_dev, bool e4m3, void* stream) {
  return guarded([&] {
    IVID_NOT_NULL(x0_dev); IVID_NOT_NULL(gamma_host); IVID_NOT_NULL(beta_host); IVID_NOT_NULL(out_fp16_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int C = C0 + (x1_dev ? C1 : 0);
    if (!x1_dev) C1 = 0;
    DevBuf dg(C * 4), dbt(C * 4), st0(static_cast<size_t>(N) * C0 * 16), st1(static_cast<size_t>(N) * std::max(C1, 1) * 16);
    IVID_CHECK_CUDA(cudaMemcpyAsync(dg.p, gamma_host, C * 4, cudaMemcpyHostToDevice, st));
    IVID_CHECK_CUDA(cudaMemcpyAsync(dbt.p, beta_host, C * 4, cudaMemcpyHostToDevice, st));
    IVID_CHECK_CUDA(cudaMemsetAsync(st0.p, 0, static_cast<size_t>(N) * C0 * 16, st));
    IVID_CHECK_CUDA(cudaMemsetAsync(st1.p, 0, static_cast<size_t>(N) * std::max(C1, 1) * 16, st));
    launch_gn_stats(x0_dev, static_cast<double*>(st0.p), N, H * W, C0, st);
    if (C1 > 0) launch_gn_stats(x1_dev, static_cast<double*>(st1.p), N, H * W, C1, st);
    GnApplyDesc g;
    g.x0 = x0_dev; g.x1 = C1 > 0 ? x1_dev : nullptr; g.C0 = C0; g.C1 = C1; g.N = N; g.H = H; g.W = W; g.mode = mode;
    g.silu = silu; g.out_act = out_fp16_dev; g.out_e4m3 = e4m3;
    g.stats0 = static_cast<double*>(st0.p); g.stats1 = C1 > 0 ? static_cast<double*>(st1.p) : nullptr;
    g.groups = groups; g.eps = eps; g.gamma = static_cast<float*>(dg.p); g.beta = static_cast<float*>(dbt.p);
    g.film = film_dev; g.film_ld = 2 * C; g.film_off = 0;
    launch_gn_apply(g, st);
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  });
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

}  // extern "C"
