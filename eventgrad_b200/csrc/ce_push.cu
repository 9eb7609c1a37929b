// eventgrad_b200 -- copy-engine push for the split step of dense gossip (decent).  sm_90a.
//
// The split step (csrc/gossip.cu, phase 1 / phase 2) hides the neighbour pushes behind forward/backward,
// but its phase-1 kernel occupies up to 128 CTAs while the 2 x 70 MB cross NVLink -- SMs and
// issue slots taken from the convolutions it overlaps with.  For `decent` every tile is pushed every step,
// so the push is a plain contiguous copy: this path hands it to the DMA engines instead,
//
//     wait_acks<<<1,32>>>      WAR guard: both neighbours consumed what was pushed at step k-1
//     cudaMemcpyAsync x 2      theta_k -> left.inbox_r, theta_k -> right.inbox_l   (peer-mapped, copy engines)
//     publish_pushed<<<1,32>>> fence.sys + st.release.sys pushed_to_{l,r} = k
//
// on the side stream, and phase 2 (wait pushed flags, mix, SGD, ack) runs unchanged.  All three are
// ordinary stream work with device-resident step numbers, so the sequence is CUDA-graph capturable.
// Opt-in: TrainConfig.ce_push (--ce-push); needs overlap_push and algo=decent.  Not yet run on hardware.
// Replaces the MPI_Issend/MPI_Recv pair of /root/reference/dmnist/decent/decent.cpp:192-208.
#include "api.h"
#include "common.cuh"

namespace egb {

__global__ void ce_wait_acks_kernel(const GossipParams p) {
  if (threadIdx.x == 0 && p.sync) {
    const uint32_t step = (uint32_t)(*p.fsm.pass_num + 1);
    wait_ge(p.ack_from_l, step - 1u, p.status, p.timeout_ns);
    wait_ge(p.ack_from_r, step - 1u, p.status, p.timeout_ns);
  }
}

__global__ void ce_publish_pushed_kernel(const GossipParams p) {
  if (threadIdx.x == 0) {
    const uint32_t step = (uint32_t)(*p.fsm.pass_num + 1);
    // the copies precede this kernel in stream order (complete and visible before it starts); the fence
    // orders them before the flags for an observer that acquires the flag at system scope
    __threadfence_system();
    st_release_sys(p.pushed_to_l, step);
    st_release_sys(p.pushed_to_r, step);
  }
}

cudaError_t launch_ce_push(const GossipParams& p, cudaStream_t s) {
  // push_r null: 2-rank ring, one copy.  Every step pushes: no --local-steps, no --global-avg-period
  if (p.push_l == nullptr || p.fsm.enabled || p.local_steps > 1 || p.global_avg_period != 0)
    return cudaErrorInvalidValue;
  const size_t nbytes = (size_t)p.tab.n_tiles * EG_TILE * sizeof(float);
  eg_count_launch(EG_FAM_GOSSIP, 2);
  ce_wait_acks_kernel<<<1, 32, 0, s>>>(p);
  cudaError_t e = cudaMemcpyAsync(p.push_l, p.theta, nbytes, cudaMemcpyDeviceToDevice, s);
  if (e != cudaSuccess) return e;
  if (p.push_r != nullptr && p.push_r != p.push_l) {
    e = cudaMemcpyAsync(p.push_r, p.theta, nbytes, cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) return e;
  }
  ce_publish_pushed_kernel<<<1, 32, 0, s>>>(p);
  return cudaGetLastError();
}

}  // namespace egb
