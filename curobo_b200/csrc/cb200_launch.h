// cb200_launch.h -- one spelling for a kernel launch, so that the host emulation build (tests/simt: the translation unit compiled
// as C++ with CB200_SIMT_EMULATION, CTA threads played by std::threads) runs the SAME launchers -- argument checks, shared-memory
// sizing, variant selection, grid sizing -- on the CPU.  Under nvcc the macro is exactly the triple-chevron launch.
// Also the host helpers every launching unit shares: error status, device properties, grid sizing, shared-memory opt-in.
#pragma once
#include <algorithm>
// CB200_EXTERN_SHARED declares a kernel's dynamic shared-memory array.  Under nvcc it is exactly `extern __shared__`; in the host
// emulation `__shared__` alone means "static" (a CTA-wide array inside a kernel), so the extern declaration needs its own spelling.
#ifdef CB200_SIMT_EMULATION
#define CB200_EXTERN_SHARED extern
#else
#define CB200_EXTERN_SHARED extern __shared__
#endif
#ifdef CB200_SIMT_EMULATION
#define CB200_LAUNCH(kernel, grid, block, smem_bytes, stream, ...) simt::launch(kernel, (int)(grid), (int)(block), __VA_ARGS__)
#else
#define CB200_LAUNCH(kernel, grid, block, smem_bytes, stream, ...) kernel<<<(grid), (block), (smem_bytes), (stream)>>>(__VA_ARGS__)
#endif

// A barrier among a SUBSET of a CTA's warps (PTX named barrier): the warps of a team that shares one row meet without the other
// teams of the CTA.  `nthreads` must be a multiple of 32; ids 1..15 (0 is __syncthreads).
#ifdef CB200_SIMT_EMULATION
#define CB200_NAMED_BARRIER(id, nthreads) simt::named_barrier((id), (nthreads))
#else
#define CB200_NAMED_BARRIER(id, nthreads) asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory")
#endif

namespace cb200 {
inline int ret(cudaError_t e) {
  if (e != cudaSuccess) (void)cudaGetLastError();  // do not leave a stale error for the caller's next CUDA call
  return (int)e;
}
inline int launch_status() { return ret(cudaGetLastError()); }

// Properties of the CURRENT device (the host layer makes the tensors' device current around every call), cached per
// ordinal: one process may drive several GPUs, and cudaFuncSetAttribute / occupancy results are per device.
struct DevInfo {
  int sm_count = 0, max_smem = 0, ordinal = 0;
  bool ok = false;
};
constexpr int kMaxDevices = 64;
inline DevInfo &dev_info() {
  static thread_local DevInfo table[kMaxDevices];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  DevInfo &d = table[dev];
  if (!d.ok) {
    d.ordinal = dev;
    cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&d.max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    d.ok = d.sm_count > 0;
  }
  return d;
}

// One wave of `kernel`: every SM filled to its occupancy (1 CTA per SM when the query fails), but no more CTAs than work items.
template <typename K>
inline int persistent_grid(K kernel, int block, size_t smem, long long work_items) {
  int per_sm = 1;
  if (ret(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, smem)) != cudaSuccess || per_sm < 1) per_sm = 1;
  return (int)std::max(std::min((long long)dev_info().sm_count * per_sm, work_items), 1LL);
}

// Grid of a grid-stride kernel: `work` CTAs, at most `per_sm_cap` per SM, at least one.
inline int capped_grid(long long work, int per_sm_cap) {
  return (int)std::max(std::min(work, (long long)dev_info().sm_count * per_sm_cap), 1LL);
}

// Lets `kernel` take `smem` bytes of dynamic shared memory (above 48 KB a launch needs this opt-in); on failure the error, cleared.
template <typename K>
inline cudaError_t opt_in_smem(K kernel, size_t smem) {
  if (smem <= 48 * 1024) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  (void)ret(e);
  return e;
}
}  // namespace cb200

// Every launching entry point runs on the device that OWNS its output buffer, whatever the caller's current device is:
// occupancy queries, cudaFuncSetAttribute(MaxDynamicSharedMemorySize) and the launch itself are per device, and the host
// layer passes raw pointers + the tensor's stream without entering a device context.  CB200_DEVICE_GUARD(ptr) looks the
// pointer's device up (cudaPointerGetAttributes: no synchronisation, legal during graph capture), switches to it when it
// differs from the current one and switches back on scope exit.
#ifdef CB200_SIMT_EMULATION
#define CB200_DEVICE_GUARD(ptr) (void)(ptr)
#else
namespace cb200 {
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(const void *p) {
    if (p == nullptr) return;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
      (void)cudaGetLastError();
      return;
    }
    if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) return;
    if (cudaGetDevice(&prev) != cudaSuccess) return;
    if (prev != at.device && cudaSetDevice(at.device) == cudaSuccess) switched = true;
  }
  ~DeviceGuard() {
    if (switched) (void)cudaSetDevice(prev);
  }
  DeviceGuard(const DeviceGuard &) = delete;
  DeviceGuard &operator=(const DeviceGuard &) = delete;
};
}  // namespace cb200
#define CB200_DEVICE_GUARD(ptr) ::cb200::DeviceGuard cb200_device_guard_(ptr)
#endif
