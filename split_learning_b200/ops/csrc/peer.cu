// Peer-memory runtime: symmetric device allocations shared across the one-process-per-GPU
// ranks of the box through CUDA IPC handles (NVLink/NVSwitch P2P), plus host-pinned "hint"
// words in a POSIX shared-memory segment so host schedulers can poll mailbox progress
// without a device round trip.  (SURVEY §5 "Distributed communication backend".)
#include <cuda_runtime.h>
#include <stdint.h>

#include "sm90.cuh"
#include <stdint.h>
#include <string.h>

extern "C" {

int slb_device_count() {
  int n = 0;
  return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0;
}
int slb_set_device(int dev) { return -static_cast<int>(cudaSetDevice(dev)); }

// plain device allocation that can be exported (cudaMalloc, not the caching allocator)
int slb_malloc(void** out, long long bytes) {
  cudaError_t e = cudaMalloc(out, static_cast<size_t>(bytes));
  if (e != cudaSuccess) return -static_cast<int>(e);
  return -static_cast<int>(cudaMemset(*out, 0, static_cast<size_t>(bytes)));
}
int slb_free(void* p) { return -static_cast<int>(cudaFree(p)); }

// A stream of our own (non-blocking).  torch.cuda.Stream() hands out 32 pooled streams per device round-robin, so in a
// process that creates more than 32 (several clients in one process, long test sessions) two *live* stage streams can be
// the same CUDA stream — and a mailbox wait of one stage then sits in front of the kernel of the other that would publish
// that flag.  high != 0: greatest priority of the device.
int slb_stream_create(void** out, int high) {
  int least = 0, greatest = 0;
  cudaDeviceGetStreamPriorityRange(&least, &greatest);
  cudaStream_t s;
  cudaError_t e = cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, high ? greatest : least);
  if (e != cudaSuccess) return -static_cast<int>(e);
  slb::slb_det(s);                        // its reduction scratch, now rather than inside a graph capture
  *out = s;
  return 0;
}
int slb_stream_destroy(void* s) {
  slb::slb_det_release(static_cast<cudaStream_t>(s));
  return -static_cast<int>(cudaStreamDestroy(static_cast<cudaStream_t>(s)));
}

int slb_ipc_get_handle(void* p, uint8_t* out64) {
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) return -static_cast<int>(e);
  static_assert(sizeof(h) == 64, "ipc handle size");
  memcpy(out64, &h, 64);
  return 0;
}
int slb_ipc_open(const uint8_t* in64, void** out) {
  cudaIpcMemHandle_t h;
  memcpy(&h, in64, 64);
  return -static_cast<int>(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
}
int slb_ipc_close(void* p) { return -static_cast<int>(cudaIpcCloseMemHandle(p)); }

int slb_can_access_peer(int dev, int peer) {
  int ok = 0;
  cudaDeviceCanAccessPeer(&ok, dev, peer);
  return ok;
}
int slb_enable_peer(int peer) {
  cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return 0; }
  return -static_cast<int>(e);
}

// map an existing host range (e.g. mmap'ed /dev/shm segment) for device access; returns device pointer
int slb_host_register(void* host, long long bytes, void** dev_ptr) {
  cudaError_t e = cudaHostRegister(host, static_cast<size_t>(bytes), cudaHostRegisterMapped | cudaHostRegisterPortable);
  if (e != cudaSuccess && e != cudaErrorHostMemoryAlreadyRegistered) return -static_cast<int>(e);
  if (e == cudaErrorHostMemoryAlreadyRegistered) cudaGetLastError();
  return -static_cast<int>(cudaHostGetDevicePointer(dev_ptr, host, 0));
}
int slb_host_unregister(void* host) { return -static_cast<int>(cudaHostUnregister(host)); }

int slb_memcpy_async(void* dst, const void* src, long long bytes, cudaStream_t st) {
  return -static_cast<int>(cudaMemcpyAsync(dst, src, static_cast<size_t>(bytes), cudaMemcpyDefault, st));
}
const char* slb_error_string(int code) { return cudaGetErrorString(static_cast<cudaError_t>(code < 0 ? -code : code)); }

}  // extern "C"
