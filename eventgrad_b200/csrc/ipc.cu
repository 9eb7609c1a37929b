// eventgrad_b200 -- CUDA-IPC window runtime: the H100-native replacement of the reference's
// MPI RMA window (MPI_Alloc_mem + MPI_Win_create, /root/reference/dmnist/event/event.cpp:170-179).
// Each rank cudaMalloc's one slab, exports a 64-byte IPC handle (exchanged through the process
// group by Python), and maps every peer's slab into its own address space.  Stores to a mapped
// peer pointer from inside a kernel are the MPI_Put; NVSwitch routes them at NVLink-5 speed.
#include "api.h"

namespace egb {

static_assert(sizeof(cudaIpcMemHandle_t) == sizeof(IpcHandle), "IPC handle size");

cudaError_t ipc_alloc(size_t nbytes, void** ptr, IpcHandle* h) {
  cudaError_t e = cudaMalloc(ptr, nbytes);
  if (e != cudaSuccess) return e;
  e = cudaMemset(*ptr, 0, nbytes);   // window starts zeroed (event.cpp:144-147)
  if (e != cudaSuccess) return e;
  e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return e;
  return cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(h), *ptr);
}

cudaError_t ipc_open(const IpcHandle& h, void** ptr) {
  cudaIpcMemHandle_t hh;
  memcpy(&hh, &h, sizeof(hh));
  return cudaIpcOpenMemHandle(ptr, hh, cudaIpcMemLazyEnablePeerAccess);
}

cudaError_t ipc_close(void* ptr) { return cudaIpcCloseMemHandle(ptr); }
cudaError_t ipc_free(void* ptr) { return cudaFree(ptr); }

}  // namespace egb
