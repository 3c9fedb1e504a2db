// Symmetric-heap fabric: every rank cudaMallocs its shard, exports a CUDA IPC handle, and maps
// all peers' shards, so kernels address any shard by pointer (NVLink/NVSwitch one-sided access).
// This replaces Flink's partitionCustom + network stack (FPS:416-420,455-463).  NCCL is used
// only to bootstrap (exchange the 64-byte handles) and for barriers.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

extern "C" int fps_heap_alloc(size_t bytes, void** out) {
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) return (int)e;
  e = cudaMemset(p, 0, bytes);
  if (e != cudaSuccess) return (int)e;
  *out = p;
  return 0;
}
extern "C" int fps_heap_free(void* p) { return (int)cudaFree(p); }

extern "C" int fps_ipc_get_handle(void* p, unsigned char* out64) {
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) return (int)e;
  memcpy(out64, &h, sizeof(h));
  return 0;
}
extern "C" int fps_ipc_open_handle(const unsigned char* in64, void** out) {
  cudaIpcMemHandle_t h;
  memcpy(&h, in64, sizeof(h));
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return (int)e;
  *out = p;
  return 0;
}
extern "C" int fps_ipc_close(void* p) { return (int)cudaIpcCloseMemHandle(p); }

// single-process multi-GPU mode (tests / notebooks): plain peer access
extern "C" int fps_enable_peer(int dev, int peer) {
  int can = 0;
  cudaError_t e = cudaDeviceCanAccessPeer(&can, dev, peer);
  if (e != cudaSuccess) return (int)e;
  if (!can) return -1;
  int cur = 0;
  cudaGetDevice(&cur);
  cudaSetDevice(dev);
  e = cudaDeviceEnablePeerAccess(peer, 0);
  cudaSetDevice(cur);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();
    return 0;
  }
  return (int)e;
}

extern "C" int fps_device_info(int dev, int* sm_count, int* cc_major, int* cc_minor,
                               size_t* total_mem) {
  cudaDeviceProp p;
  cudaError_t e = cudaGetDeviceProperties(&p, dev);
  if (e != cudaSuccess) return (int)e;
  *sm_count = p.multiProcessorCount;
  *cc_major = p.major;
  *cc_minor = p.minor;
  *total_mem = p.totalGlobalMem;
  return 0;
}
extern "C" const char* fps_error_string(int code) {
  if (code == -1000) return "dim too large for fused kernel";
  if (code == -1001) return "unsupported id width";
  if (code == -1009) return "row-wise AdaGrad does not support this kernel variant";
  if (code < 0) return "fps: invalid argument";
  return cudaGetErrorString((cudaError_t)code);
}
