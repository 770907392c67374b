"""python scripts/bench_pooled_dense.py

Cost of pooled dense mass windows (DenseMassMatrixTuner with rn_config.adaptation = RN_ADAPT_POOLED) against per-chain dense
windows, one GPU, two workloads:
  * eight schools, DefaultConfig with DenseMassMatrixTuner(50, 1.5, 50, 50), 8192 chains, thread-per-chain shape;
  * funnel(60), HMC(10) with DenseMassMatrixTuner(50, 1.5, 50, 50), 1024 chains, warp-per-chain shape (n = 60 > L = 50:
    each chain's own first window covariance is rank-deficient, so the per-chain run's matrices are not usable; it is timed
    for the cost only).
Warmup is device-timed with CUDA events on the sampler's stream (the second run of each mode; the first compiles its kernels).
A separate profiled run (torch.profiler, CUDA activities) of each pooled warmup sums the device time of the window-end kernels
(rn_k_pool_reduce, rn_k_pool_reduce_dense, rn_k_pool_factor, rn_k_pool_apply_dense) and divides by the windows closed.
Prints one JSON line with the card and its power limit."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle.rainier_py import configs  # noqa: E402
from rainier_b200 import abi, api  # noqa: E402

WINDOW_KERNELS = ("rn_k_pool_reduce", "rn_k_pool_reduce_dense", "rn_k_pool_factor", "rn_k_pool_apply_dense")


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def windows_closed(config):
    cfg, keep = api.lower_config(config)
    size, i, out = cfg.initial_window_size, 0, 0
    for j in range(1, cfg.warmup_iterations + 1):
        if j < cfg.skip_first or (cfg.warmup_iterations - j) < cfg.skip_last:
            continue
        i += 1
        if i == size:
            out, i, size = out + 1, 0, int(size * cfg.window_expansion)
    return out


def warmup_ms(model, config, seeds):
    s = api.CudaSampler(model, config, seeds=seeds)
    stream = torch.cuda.ExternalStream(s.stream, device=torch.device("cuda", 0))
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record(stream)
    s.warmup(-1)
    ev[1].record(stream)
    s.sync()
    torch.cuda.synchronize()
    s.close()
    return ev[0].elapsed_time(ev[1])


def window_end_us(model, config, seeds):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s = api.CudaSampler(model, config, seeds=seeds)
        s.warmup(-1)
        s.sync()
        s.close()
        torch.cuda.synchronize()
    per = {k: 0.0 for k in WINDOW_KERNELS}
    for e in prof.events():
        if e.name in per:
            per[e.name] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    w = windows_closed(config)
    return {k: v / w for k, v in per.items()}, sum(per.values()) / w, w


def workload(name, rir, cols, config_for, chains, backend):
    model = api.CudaModel(rir, cols, device=0)
    seeds = np.arange(chains, dtype=np.int64) + 1
    out = {"chains": chains, "backend": "thread" if backend == abi.RN_BACKEND_THREAD else "warp"}
    for mode, adaptation in (("per_chain_dense", abi.RN_ADAPT_PER_CHAIN), ("pooled_dense", abi.RN_ADAPT_POOLED)):
        config = config_for(adaptation, backend)
        warmup_ms(model, config, seeds)  # compiles the module
        out[mode + "_warmup_ms"] = [warmup_ms(model, config, seeds) for _ in range(2)]
    per, total, w = window_end_us(model, config_for(abi.RN_ADAPT_POOLED, backend), seeds)
    out.update({"windows": w, "window_end_device_us": total, "window_end_device_us_by_kernel": per})
    model.close()
    return name, out


def schools_config(adaptation, backend):
    c = api.SamplerConfig(iterations=1, warmupIterations=500, adaptation=adaptation, backend=backend)
    c._massMatrixTuner = api.DenseMassMatrixTuner(50, 1.5, 50, 50)
    return c


def funnel_config(adaptation, backend):
    return api.make_config(iterations=1, warmupIterations=500, sampler=api.HMCSampler(10), stepSizeTuner=api.DualAvgTuner(0.8),
                           massMatrixTuner=api.DenseMassMatrixTuner(50, 1.5, 50, 50), adaptation=adaptation, backend=backend)


def main():
    torch.cuda.set_device(0)
    res = {}
    rir, cols = configs.eight_schools().compile(True)
    k, v = workload("eight_schools", rir, cols, schools_config, 8192, abi.RN_BACKEND_THREAD)
    res[k] = v
    rir, cols = configs.funnel(60).compile(True)
    k, v = workload("funnel60", rir, cols, funnel_config, 1024, abi.RN_BACKEND_WARP)
    res[k] = v
    print(json.dumps(dict(res, warmup_iterations=500, gpu=card())), flush=True)


if __name__ == "__main__":
    main()
