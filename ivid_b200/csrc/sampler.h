// DDPM / DDIM / DPM-Solver++ samplers (host class).  See sampler.cu / sampler.cuh.
#pragma once
#include <vector>

#include "unet.h"

namespace ivid {

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
  // the whole reverse process
  void run(Unet& unet, float* x, int N, int steps, const ivid_step_args_t& a, const float* noise_all,
           const float* cond_noise_all, float* traj_x0, float* traj_xt, cudaStream_t stream);

 private:
  void ensure_device(int N2, size_t eps_elems);
  void ensure_hist(size_t elems);
  int T_;
  std::vector<double> betas_, acp_, acp_prev_, srac_, srm1_, pvar_, plogvar_, pc1_, pc2_;
  void* d_table_ = nullptr;
  void* d_state_ = nullptr;
  double* d_acp_ = nullptr;                // float64 alphas_cumprod (DPM-Solver++ step scalars)
  float* d_hist_ = nullptr;                // DPM-Solver++ history D_{-1} [N,C,H,W], updated in place by the step kernels
  size_t cap_hist_ = 0;
  int64_t* d_t_ = nullptr;
  int64_t* d_classes2_ = nullptr;
  float* d_eps_ = nullptr;
  float* d_xtmp_ = nullptr;
  bool no_fuse_ = false;                   // inside run() with per-step noise / trajectory pointers: keep the separate step kernel
  bool classes2_ready_ = false;            // d_classes2_ already holds [classes, -1 ...] for (classes2_src_, classes2_n_)
  const int64_t* classes2_src_ = nullptr;
  int classes2_n_ = 0;
  int cap_n_ = 0;
  size_t cap_eps_ = 0;
};

}  // namespace ivid
