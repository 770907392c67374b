// tests/pool_probe.cu -- TEST INFRASTRUCTURE ONLY: launches the pooled mass-window kernels (rn_k_pool_reduce,
// rn_k_pool_apply) of a module the runtime emitted (CudaModel.emit_cubin) on crafted chain statistics, with the grid and
// block shapes of rn_runtime.cpp's pool_window.  It holds no kernel logic: the module is loaded as it is, and the passes
// and the emulated all-reduce over ranks are orchestrated by tests/test_gpu_pooled_mass.py.
#include <cuda.h>

#include <cstring>

#include "../rainier_b200/csrc/rn_args.h"

extern "C" {

// loads a cubin into the device's primary context (the one torch uses); returns a CUresult
int pool_probe_load(const void* cubin, int device, void** mod_out) {
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

int pool_probe_unload(void* mod, int device) {
  CUdevice dev;
  CUresult r = cuModuleUnload((CUmodule)mod);
  if (r == CUDA_SUCCESS) r = cuDeviceGet(&dev, device);
  if (r == CUDA_SUCCESS) r = cuDevicePrimaryCtxRelease(dev);
  return (int)r;
}

// one launch on one emulated rank's chains, then a synchronisation; which 0: rn_k_pool_reduce(pass) on n blocks of 256
// threads, 1: rn_k_pool_apply on ceil(chains / 128) blocks of 128.  The arrays are that rank's [field][chains] device
// arrays; the RnArgs fields the two kernels do not read stay zero.
int pool_probe_launch(void* mod, int which, int n, int chains, double* est_mean, double* est_raw, double* mass, double* da,
                      int* da_iter, int* st_err, int step_tuner, double* pool, int window_len, int pass) {
  RnArgs a;
  std::memset(&a, 0, sizeof(a));
  a.chains = chains;
  a.est_mean = est_mean;
  a.est_raw = est_raw;
  a.mass = mass;
  a.da = da;
  a.da_iter = da_iter;
  a.st_err = st_err;
  a.step_tuner = step_tuner;
  CUfunction f;
  CUresult r = cuModuleGetFunction(&f, (CUmodule)mod, which ? "rn_k_pool_apply" : "rn_k_pool_reduce");
  if (r != CUDA_SUCCESS) return (int)r;
  CUdeviceptr p = (CUdeviceptr)pool;
  int wl = window_len, ps = pass;
  if (which == 0) {
    void* params[] = {&a, &p, &wl, &ps};
    r = cuLaunchKernel(f, (unsigned)n, 1, 1, 256, 1, 1, 0, nullptr, params, nullptr);
  } else {
    void* params[] = {&a, &p, &wl};
    r = cuLaunchKernel(f, (unsigned)((chains + 127) / 128), 1, 1, 128, 1, 1, 0, nullptr, params, nullptr);
  }
  if (r == CUDA_SUCCESS) r = cuCtxSynchronize();
  return (int)r;
}

}  // extern "C"
