// tests/diag_probe.cu -- TEST INFRASTRUCTURE ONLY: launches the tracked-diagnostics kernels (rn_k_diag_accum,
// rn_k_diag_terms, rn_k_diag_reduce) of a module the runtime emitted (CudaModel.emit_cubin) with the grid and block shapes
// of rn_runtime.cpp's track_accumulate and rn_sampler_tracked_diagnostics, on one emulated rank's chain block.  It holds no
// kernel logic: the passes and the emulated all-reduce over ranks are orchestrated by tests/test_gpu_tracked_diagnostics_ranks.py.
#include <cuda.h>

extern "C" {

// loads a cubin into the device's primary context (the one torch uses); returns a CUresult
int diag_probe_load(const void* cubin, int device, void** mod_out) {
  CUdevice dev;
  CUcontext ctx;
  CUresult r = cuInit(0);
  if (r == CUDA_SUCCESS) r = cuDeviceGet(&dev, device);
  if (r == CUDA_SUCCESS) r = cuDevicePrimaryCtxRetain(&ctx, dev);
  if (r == CUDA_SUCCESS) r = cuCtxSetCurrent(ctx);
  CUmodule mod = nullptr;
  if (r == CUDA_SUCCESS) r = cuModuleLoadData(&mod, cubin);
  *mod_out = mod;
  return (int)r;
}

int diag_probe_unload(void* mod, int device) {
  CUdevice dev;
  CUresult r = cuModuleUnload((CUmodule)mod);
  if (r == CUDA_SUCCESS) r = cuDeviceGet(&dev, device);
  if (r == CUDA_SUCCESS) r = cuDevicePrimaryCtxRelease(dev);
  return (int)r;
}

// rn_k_diag_accum on ceil(C / threads) x n blocks of `threads`, (99 + sub) * threads doubles of dynamic shared memory
int diag_probe_accum(void* mod, const double* draws, int n, int C, int j0, int thin, int m, long long T0, int sub, double* state,
                     int threads) {
  CUfunction f;
  CUresult r = cuModuleGetFunction(&f, (CUmodule)mod, "rn_k_diag_accum");
  const int smem = (99 + sub) * threads * 8;
  if (r == CUDA_SUCCESS) r = cuFuncSetAttribute(f, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, smem);
  CUdeviceptr s = (CUdeviceptr)draws, st = (CUdeviceptr)state;
  void* params[] = {&s, &n, &C, &j0, &thin, &m, &T0, &sub, &st};
  if (r == CUDA_SUCCESS)
    r = cuLaunchKernel(f, (unsigned)((C + threads - 1) / threads), (unsigned)n, 1, (unsigned)threads, 1, 1, (unsigned)smem, nullptr,
                       params, nullptr);
  if (r == CUDA_SUCCESS) r = cuCtxSynchronize();
  return (int)r;
}

// rn_k_diag_terms on ceil(C / 128) x n blocks of 128
int diag_probe_terms(void* mod, const double* state, int n, int C, long long T, int L, int q0, int nq, double* out) {
  CUfunction f;
  CUresult r = cuModuleGetFunction(&f, (CUmodule)mod, "rn_k_diag_terms");
  CUdeviceptr st = (CUdeviceptr)state, o = (CUdeviceptr)out;
  void* params[] = {&st, &n, &C, &T, &L, &q0, &nq, &o};
  if (r == CUDA_SUCCESS)
    r = cuLaunchKernel(f, (unsigned)((C + 127) / 128), (unsigned)n, 1, 128, 1, 1, 0, nullptr, params, nullptr);
  if (r == CUDA_SUCCESS) r = cuCtxSynchronize();
  return (int)r;
}

// rn_k_diag_reduce on `rows` blocks of 256 (shift may be NULL)
int diag_probe_reduce(void* mod, const double* in, int rows, int C, const double* shift, double* out) {
  CUfunction f;
  CUresult r = cuModuleGetFunction(&f, (CUmodule)mod, "rn_k_diag_reduce");
  CUdeviceptr i = (CUdeviceptr)in, sh = (CUdeviceptr)shift, o = (CUdeviceptr)out;
  void* params[] = {&i, &C, &sh, &o};
  if (r == CUDA_SUCCESS) r = cuLaunchKernel(f, (unsigned)rows, 1, 1, 256, 1, 1, 0, nullptr, params, nullptr);
  if (r == CUDA_SUCCESS) r = cuCtxSynchronize();
  return (int)r;
}

}  // extern "C"
