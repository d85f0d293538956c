// oracle/ref_legacy_trajectory_launcher.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.
//
// Thin extern "C" launchers around the REFERENCE's legacy trajectory kernels -- the POSITION (clique) and ACCELERATION
// control spaces -- #included from the reference tree where they lie (-I <reference>/curobo/_src/curobolib/kernels; nothing is
// copied into this repository).  Built by curobo_b200/build.py::build_reference_legacy_kernels into
// oracle/_ref/libcurobo_ref_legacy.so (git-ignored; travels to the GPU box with the snapshot).  Used ONLY by
// tests/ref_legacy_kernels.py to compare our kernels with the reference's on the same inputs.
//
// Launch math follows backends/pybind/trajectory_kernel_launch.cu:26-107 (forward, 128 threads over batch*dof*horizon),
// :110-178 (backward, 128 threads over batch*dof*(horizon-4)), :181-254 (integration, 512 threads over batch*dof).  The
// integration kernel is templated on the horizon (the cuda.core backend JIT-compiles it per horizon,
// cuda_core_backend/trajectory.py:495-505): the horizons the tests use are instantiated.
#include <cstdint>
#include <cuda_runtime.h>

#include "trajectory/legacy/differentiation_position_kernel.cuh"
#include "trajectory/legacy/integration_acceleration_kernel.cuh"

namespace clg = curobo::trajectory::legacy;

extern "C" {

int ref_clique_forward(float *op, float *ov, float *oa, float *oj, float *odt, const float *u, const float *sp,
                       const float *sv, const float *sa, const float *gp, const float *gv, const float *ga,
                       const int32_t *sidx, const int32_t *gidx, const float *traj_dt, const uint8_t *implicit, int B,
                       int H, int D, cudaStream_t stream) {
  const int k_size = B * D * H;
  const int threads = k_size > 128 ? 128 : k_size;
  const int blocks = (k_size + threads - 1) / threads;
  clg::position_clique_loop_idx_fwd_kernel<float, true><<<blocks, threads, 0, stream>>>(
      op, ov, oa, oj, odt, u, sp, sv, sa, gp, gv, ga, sidx, gidx, traj_dt, implicit, B, H, D);
  return (int)cudaGetLastError();
}

int ref_clique_backward(float *out, const float *gp, const float *gv, const float *ga, const float *gj, const float *traj_dt,
                        const int32_t *dt_idx, const uint8_t *implicit, int B, int H, int D, cudaStream_t stream) {
  const int k_size = B * D * (H - 4);
  const int threads = k_size > 128 ? 128 : k_size;
  const int blocks = (k_size + threads - 1) / threads;
  clg::position_clique_loop_idx_bwd_kernel<float, true><<<blocks, threads, 0, stream>>>(
      out, gp, gv, ga, gj, traj_dt, dt_idx, implicit, B, H, D);
  return (int)cudaGetLastError();
}

int ref_integrate_acceleration(float *op, float *ov, float *oa, float *oj, const float *u, const float *sp, const float *sv,
                               const float *sa, const int32_t *sidx, const float *traj_dt, int B, int H, int D,
                               cudaStream_t stream) {
  const int k_size = B * D;
  const int threads = k_size > 512 ? 512 : k_size;
  const int blocks = (k_size + threads - 1) / threads;
#define CB_ACC(HH)                                                                                                         \
  if (H == HH) {                                                                                                           \
    clg::acceleration_loop_idx_rk2_kernel<float, HH><<<blocks, threads, 0, stream>>>(op, ov, oa, oj, u, sp, sv, sa, sidx, \
                                                                                     traj_dt, B, H, D);                   \
    return (int)cudaGetLastError();                                                                                        \
  }
  CB_ACC(8)
  CB_ACC(9)
  CB_ACC(14)
  CB_ACC(30)
  CB_ACC(34)
#undef CB_ACC
  return -1;
}

}  // extern "C"
