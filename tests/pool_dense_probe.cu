// tests/pool_dense_probe.cu -- TEST INFRASTRUCTURE ONLY: launches the pooled dense mass-window kernels (rn_k_pool_reduce
// pass 0, rn_k_pool_reduce_dense, rn_k_pool_factor, rn_k_pool_apply_dense) of a module the runtime emitted
// (CudaModel.emit_cubin) on crafted chain statistics, with the grid and block shapes of rn_runtime.cpp's pool_window_dense.
// It holds no kernel logic: the module is loaded as it is (pool_probe_load / pool_probe_unload of the same shape as
// tests/pool_probe.cu), and the passes and the emulated all-reduce over ranks are orchestrated by
// tests/test_gpu_pooled_dense.py.
#include <cuda.h>

#include <algorithm>
#include <cstring>

#include "../rainier_b200/csrc/rn_args.h"

extern "C" {

int pool_dense_probe_load(const void* cubin, int device, void** mod_out) {
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

int pool_dense_probe_unload(void* mod, int device) {
  CUdevice dev;
  CUresult r = cuModuleUnload((CUmodule)mod);
  if (r == CUDA_SUCCESS) r = cuDeviceGet(&dev, device);
  if (r == CUDA_SUCCESS) r = cuDevicePrimaryCtxRelease(dev);
  return (int)r;
}

// one launch on one emulated rank's chains, then a synchronisation.  which 0: rn_k_pool_reduce(pass 0) on n blocks of 256,
// 1: rn_k_pool_reduce_dense on n^2 blocks of 256, 2: rn_k_pool_factor on one block of min(512, n rounded up to 32),
// 3: rn_k_pool_apply_dense on ceil(chains / 128) x min(n, 64) blocks of 128.  The arrays are that rank's [field][chains]
// device arrays; the RnArgs fields the kernels do not read stay zero.
int pool_dense_probe_launch(void* mod, int which, int n, int chains, double* est_mean, double* est_raw, double* est_cov,
                            double* mass, double* chol, double* da, int* da_iter, int* st_err, int step_tuner, double* pool,
                            int window_len) {
  RnArgs a;
  std::memset(&a, 0, sizeof(a));
  a.chains = chains;
  a.est_mean = est_mean;
  a.est_raw = est_raw;
  a.est_cov = est_cov;
  a.mass = mass;
  a.chol = chol;
  a.da = da;
  a.da_iter = da_iter;
  a.st_err = st_err;
  a.step_tuner = step_tuner;
  static const char* names[] = {"rn_k_pool_reduce", "rn_k_pool_reduce_dense", "rn_k_pool_factor", "rn_k_pool_apply_dense"};
  CUfunction f;
  CUresult r = cuModuleGetFunction(&f, (CUmodule)mod, names[which]);
  if (r != CUDA_SUCCESS) return (int)r;
  CUdeviceptr p = (CUdeviceptr)pool;
  int wl = window_len, pass = 0;
  if (which == 0) {
    void* params[] = {&a, &p, &wl, &pass};
    r = cuLaunchKernel(f, (unsigned)n, 1, 1, 256, 1, 1, 0, nullptr, params, nullptr);
  } else if (which == 1) {
    void* params[] = {&a, &p, &wl};
    r = cuLaunchKernel(f, (unsigned)(n * n), 1, 1, 256, 1, 1, 0, nullptr, params, nullptr);
  } else if (which == 2) {
    void* params[] = {&p, &wl};
    r = cuLaunchKernel(f, 1, 1, 1, (unsigned)std::min(512, (n + 31) / 32 * 32), 1, 1, 0, nullptr, params, nullptr);
  } else {
    void* params[] = {&a, &p, &wl};
    r = cuLaunchKernel(f, (unsigned)((chains + 127) / 128), (unsigned)std::min(n, 64), 1, 128, 1, 1, 0, nullptr, params, nullptr);
  }
  if (r == CUDA_SUCCESS) r = cuCtxSynchronize();
  return (int)r;
}

}  // extern "C"
