// DDPM / DDIM / DPM-Solver++ / UniPC samplers (host class).  See sampler.cu / sampler.cuh.
#pragma once
#include <vector>

#include "unet.h"

namespace ivid {

struct StepPlan;   // what one step runs (sampler.cu)
struct ApgParams;  // the planes and parameters of an APG step (sampler.cuh)

class Sampler {
 public:
  Sampler(const double* betas, int T);
  ~Sampler();
  int timesteps() const { return T_; }
  const std::vector<double>& table(int which) const;

  // one reverse step (sample_once).  stream_id = Philox stream for in-kernel noise.
  // t_dev / t_prev_dev (optional): read the step from element 0 of device tensors instead of the host ints
  void step(Unet& unet, const float* x_t, float* x_prev, float* pred_x0, int N, int t, int t_prev,
            const ivid_step_args_t& a, int stream_id, cudaStream_t stream, const int64_t* t_dev = nullptr,
            const int64_t* t_prev_dev = nullptr);
  // q(x_t | x_0) of the reference's step minus 1 t over N * per_sample elements; noise == nullptr draws Philox(seed)
  void diffuse(const float* x0, const float* noise, int N, size_t per_sample, int t, uint64_t seed, float* out,
               cudaStream_t stream) const;
  // the whole reverse process (a.start_step: from that step of the grid on)
  void run(Unet& unet, float* x, int N, int steps, const ivid_step_args_t& a, const float* noise_all,
           const float* cond_noise_all, float* traj_x0, float* traj_xt, cudaStream_t stream);

 private:
  void check_step_args(const ivid_step_args_t& a, const Unet& unet, int N) const;
  // one step of checked arguments.  allow_fuse: the update may run as the output head's last kernel; classes2_filled:
  // d_classes2_ already holds [classes, -1 ...] of a.classes_dev and N
  void step_impl(Unet& unet, const float* x_t, float* x_prev, float* pred_x0, int N, const StepPlan& sp,
                 const ivid_step_args_t& a, int stream_id, cudaStream_t stream, const int64_t* t_dev,
                 const int64_t* t_prev_dev, bool allow_fuse, bool classes2_filled);
  void ensure_device(int N2, size_t eps_elems);
  void ensure_hist(size_t elems);
  // APG planes and scalars for samples of img = N*C*H*W elements (sampler.cu: kApgPlanes); the buffer moves only when img
  // changes or N outgrows it
  void ensure_apg(size_t img, int N);
  ApgParams apg_params(const ivid_step_args_t& a) const;
  int T_;
  std::vector<double> betas_, acp_, acp_prev_, srac_, srm1_, pvar_, plogvar_, pc1_, pc2_;
  void* d_table_ = nullptr;
  void* d_state_ = nullptr;
  double* d_acp_ = nullptr;                // float64 alphas_cumprod (DPM-Solver++ step scalars)
  float* d_hist_ = nullptr;                // DPM-Solver++ history D_{-1} [N,C,H,W], or UniPC's history and base (4 planes),
                                           // updated in place by the step kernels
  size_t cap_hist_ = 0;
  int64_t* d_t_ = nullptr;
  int64_t* d_classes2_ = nullptr;
  float* d_thr_s_ = nullptr;               // dynamic thresholding: s of every sample [cap_n_]
  float* d_apg_ = nullptr;                 // adaptive projected guidance: D_c, m, the PAG term and the scalars
  size_t cap_apg_ = 0, apg_img_ = 0;
  float* d_eps_ = nullptr;
  float* d_xtmp_ = nullptr;
  int cap_n_ = 0;
  size_t cap_eps_ = 0;
};

}  // namespace ivid
