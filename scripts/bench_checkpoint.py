"""python scripts/bench_checkpoint.py [--small]

Wall time and bandwidth of rn_sampler_save / rn_sampler_restore on one GPU, two workloads:
  * eight schools, DefaultConfig (EHMC ring of 100, diagonal mass), 65 536 chains, tracked diagnostics at thin 1
    (201 doubles per parameter and chain);
  * cfg 5 (Poisson GLMM, 1003 parameters, 1M rows; build/models/cfg5_primal.npz when build() made it), 4096 chains.
Each sampler runs a few warmup and sampling iterations, then is saved into page-locked memory (rn_host_alloc: one DMA per
chunk) and into pageable memory (the pinned staging ring), and restored from each.  Times are host wall clock around the
blocking calls (save and restore synchronise); GB/s is blob bytes over that time.  The best of 3 repetitions after one warm
call (module load, staging allocation).  The restored sampler's re-save is checked to be the same bytes.  Prints one JSON
line with the card, its power limit and its SM clock.  --small: 4096 chains and the 100-group cfg 5 (a rehearsal)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle.rainier_py import configs  # noqa: E402
from rainier_b200 import api  # noqa: E402

REPS = 3
small = "--small" in sys.argv


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def best(fn):
    fn()
    t = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return min(t)


def measure(name, model, config, chains, track):
    s = api.CudaSampler(model, config, seeds=np.arange(chains) + 1)
    s.warmup(-1)
    if track:
        s.track_diagnostics(1)
    s.run(config.iterations)
    s.sync()
    blob = s.save()
    size = len(blob)
    out = {"workload": name, "chains": chains, "n": model.nVars, "blob_bytes": size,
           "record_bytes": api.checkpoint_info(blob)["record_bytes"]}
    pinned = api.PinnedBuffer((size,), dtype=np.uint8)
    pageable = np.empty(size, dtype=np.uint8)
    for label, buf in (("pinned", pinned.array), ("pageable", pageable)):
        secs = best(lambda: s.save(out=buf))
        out["save_%s_s" % label] = round(secs, 4)
        out["save_%s_GBps" % label] = round(size / secs / 1e9, 2)

        times = []
        for k in range(REPS + 1):  # (the first restore is the warm call)
            t0 = time.perf_counter()
            r = api.CudaSampler.restore(model, config, buf)
            times.append(time.perf_counter() - t0)
            if k < REPS:
                r.close()
        secs = min(times[1:])
        out["restore_%s_s" % label] = round(secs, 4)
        out["restore_%s_GBps" % label] = round(size / secs / 1e9, 2)
        assert bytes(r.save()) == bytes(blob), "the restored sampler's state differs"
        r.close()
    s.close()
    pinned.close()
    return out


def cfg5_model():
    g, n_obs = (100, 100000) if small else (1000, 1000000)
    f = os.path.join(ROOT, "build", "models", "cfg5_primal%s.npz" % ("_small" if small else ""))
    if os.path.exists(f):
        z = np.load(f)
        rir, cols = z["rir"].tobytes(), [z["c%d" % i] for i in range(int(z["ncols"]))]
    else:
        rir, cols = configs.poisson_glm(g, n_obs).compile(False)
    return api.CudaModel(rir, cols), "poisson GLMM %d groups, %d obs" % (g, n_obs)


def main():
    torch.zeros(1, device="cuda")
    res = {"card": card(), "workloads": []}
    rir, cols = configs.eight_schools().compile(True)
    res["workloads"].append(measure("eight schools DefaultConfig, tracked thin 1", api.CudaModel(rir, cols),
                                    api.SamplerConfig(iterations=10, warmupIterations=20), 4096 if small else 65536, True))
    model, label = cfg5_model()
    config = api.make_config(iterations=2, warmupIterations=3, sampler=api.HMCSampler(5), stepSizeTuner=api.DualAvgTuner(0.8),
                             massMatrixTuner=api.IdentityMassMatrixTuner())
    res["workloads"].append(measure("cfg 5: " + label, model, config, 4096, False))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
