"""python scripts/bench_tracked_diagnostics.py

Cost of tracked diagnostics (rn_sampler_track_diagnostics) against the block path (rn_sampler_diagnostics over a resident
[iterations][n][chains] block), one GPU, two workloads:
  * funnel(10), HMC(5), 65 536 chains;
  * eight schools, DefaultConfig (EHMC + diagonal mass), 8192 chains.
Each runs 200 warmup and 1000 sampling iterations, thin 1.  Times are CUDA events on the sampler's stream: sampling with
tracking off (draws written to a block) and on (no block), the block path's diagnostics call, and the tracked finish.  The
accumulation time per kept draw is (sampling with tracking on - off) / 1000.  Device memory is reported for both paths: at
1000 iterations the tracker's scratch for one launch's draws is as large as the block (launch_iterations = 0 means 1000).
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
from rainier_b200 import api  # noqa: E402

ITERS = 1000


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def timed(stream, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1)


def measure(name, model, config, chains):
    n = model.nVars
    seeds = np.arange(chains) + 1
    out = {"workload": name, "chains": chains, "n": n, "iterations": ITERS}
    # tracking off: the draws go to a resident block, then the block path
    s = api.CudaSampler(model, config, seeds=seeds)
    st = torch.cuda.ExternalStream(s.stream)
    d = torch.empty((ITERS, n, chains), dtype=torch.float64, device="cuda")
    s.warmup(-1)
    out["sampling_off_ms"] = timed(st, lambda: s.run(ITERS, d.data_ptr()))
    s.diagnostics(d.data_ptr(), ITERS)  # (first call: scratch allocation)
    out["block_diagnostics_ms"] = timed(st, lambda: s.diagnostics(d.data_ptr(), ITERS))
    block = s.diagnostics(d.data_ptr(), ITERS)
    s.close()
    del d
    # tracking on, no block
    s = api.CudaSampler(model, config, seeds=seeds)
    st = torch.cuda.ExternalStream(s.stream)
    s.warmup(-1)
    s.track_diagnostics(1)
    out["sampling_on_ms"] = timed(st, lambda: s.run(ITERS, None))
    out["tracked_finish_ms"] = timed(st, lambda: s.tracked_diagnostics())
    tracked = s.tracked_diagnostics()
    s.close()
    out["accumulate_us_per_kept_draw"] = (out["sampling_on_ms"] - out["sampling_off_ms"]) * 1e3 / ITERS
    # device memory of the two paths: the tracker's state + finish scratch (8 doubles per pair) + one launch's draws when
    # rn_sampler_run gets no sample block (launch_iterations, default 1000); the block path's sample block
    launch = config.launchIterations or 1000
    out["tracked_bytes"] = {"state": 201 * 8 * n * chains, "finish_scratch": 8 * 8 * n * chains,
                            "launch_draws": 8 * min(launch, ITERS) * n * chains}
    out["block_bytes"] = 8 * ITERS * n * chains
    out["max_rel_diff_vs_block"] = float(np.max(np.abs(tracked - block) / np.maximum(np.abs(block), 1e-12)))
    return out


def main():
    torch.zeros(1, device="cuda")
    res = {"card": card(), "workloads": []}
    rir, cols = configs.funnel(10).compile(True)
    res["workloads"].append(measure("funnel10 HMC(5)", api.CudaModel(rir, cols), api.HMC(200, ITERS, 5), 65536))
    rir, cols = configs.eight_schools().compile(True)
    res["workloads"].append(measure("eight schools DefaultConfig", api.CudaModel(rir, cols),
                                    api.SamplerConfig(iterations=ITERS, warmupIterations=200), 8192))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
