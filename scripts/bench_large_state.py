"""Cost of the per-chain state placements of the warp-per-chain sampler (RN_WPC_PLACE, rn_sampler_wpc.cuh) on one GPU.
cfg 5's Poisson GLMM (configs.poisson_glm(G, 2G), primal RIR, HMC nSteps=5, static step size, identity mass):

  * G = 1 000 fits shared memory (placement 0): P0 against forced P1 in one process, alternating, same seeds; the samples of
    P1 are compared with P0's.
  * G = 6 000 (placement 1 by itself) and, with --g16000, G = 16 000: leapfrog steps x chains / s at 1 024 and 4 096 chains.

Rates are device-timed rn_sampler_run calls (CUDA events).  The card's name and power limit are read in the same run and
printed with the numbers.  Models are cached under build/models/ like scripts/bench_configs.py (building the G = 6 000 RIR in
the Python oracle takes about a minute, G = 16 000 several).  Writes one JSON line per measurement.
Usage: python scripts/bench_large_state.py [--g16000] [--iters N] [--reps R]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from oracle.rainier_py import configs
from rainier_b200 import api


def _arg(name, default):
    for a in sys.argv:
        if a.startswith(name + "="):
            return int(a.split("=")[1])
    return default


ITERS = _arg("--iters", 20)
REPS = _arg("--reps", 3)


def cached(name, build):
    d = os.path.join(ROOT, "build", "models")
    os.makedirs(d, exist_ok=True)
    f = os.path.join(d, name + ".npz")
    if os.path.exists(f):
        z = np.load(f)
        return z["rir"].tobytes(), [z["c%d" % i] for i in range(int(z["ncols"]))]
    rir, cols = build()
    np.savez(f, rir=np.frombuffer(rir, dtype=np.uint8), ncols=len(cols), **{"c%d" % i: np.asarray(c, dtype=np.float64) for i, c in enumerate(cols)})
    return rir, cols


def glmm(g):
    return cached("glmm_%d_primal" % g, lambda: configs.poisson_glm(g, 2 * g).compile(False))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return {"card": q or torch.cuda.get_device_name(0)}


class Run:
    """One sampler compiled with RN_WPC_PLACE=place (None: the sizes decide), warmed up and run once for its outputs."""

    def __init__(self, rir, cols, chains, place):
        if place is None:
            os.environ.pop("RN_WPC_PLACE", None)
        else:
            os.environ["RN_WPC_PLACE"] = str(place)
        self.cfg = api.make_config(iterations=ITERS, warmupIterations=0, sampler=api.HMCSampler(5),
                                   stepSizeTuner=api.StaticStepSize(0.002), massMatrixTuner=api.IdentityMassMatrixTuner())
        self.model = api.CudaModel(rir, cols)
        self.src = self.model.emit_source(self.cfg)
        self.s = api.CudaSampler(self.model, self.cfg, seeds=np.arange(chains) + 1000)
        os.environ.pop("RN_WPC_PLACE", None)
        self.place = int(self.src.split("#define RN_WPC_PLACE ")[1].split()[0])
        self.k = int(self.src.split("#define RN_WPC_K ")[1].split()[0])
        self.tma = int(self.src.split("#define RN_TMA_STAGES ")[1].split()[0])
        self.s.warmup(-1)
        self.stream = torch.cuda.ExternalStream(self.s.stream)
        self.d = torch.empty((ITERS, self.model.nVars, chains), dtype=torch.float64, device="cuda")
        self.s.run(ITERS, self.d.data_ptr())
        self.s.sync()
        self.first = self.d.cpu().numpy()
        self.steps0 = sum(x.leapfrogSteps for x in self.s.stats()[0])
        self.times = []

    def time_once(self):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(self.stream)
        self.s.run(ITERS, self.d.data_ptr())
        e1.record(self.stream)
        self.s.sync()
        self.times.append(e0.elapsed_time(e1) * 1e-3)

    def rate(self):
        steps = (sum(x.leapfrogSteps for x in self.s.stats()[0]) - self.steps0) / len(self.times)
        return steps / min(self.times)

    def close(self):
        self.s.close()
        self.model.close()


def compare(label, g, chains, places):
    rir, cols = glmm(g)
    runs = [Run(rir, cols, chains, p) for p in places]
    for _ in range(REPS):  # alternate the placements so that drift on the shared host hits them alike
        for r in runs:
            r.time_once()
    base = runs[0]
    for r in runs:
        rel = float(np.max(np.abs(r.first - base.first) / np.maximum(np.abs(base.first), 1e-9)))
        print(json.dumps(dict(card(), bench=label, groups=g, n=g + 3, chains=chains, forced=places[runs.index(r)], place=r.place, wpc_k=r.k,
                              tma_stages=r.tma, iters=ITERS, best_s=round(min(r.times), 5), spread=round(max(r.times) / min(r.times) - 1, 4),
                              steps_chains_per_s=r.rate(), rel_vs_first=rel)), flush=True)
    for r in runs:
        r.close()


if __name__ == "__main__":
    compare("glmm1000_placements", 1000, 4096, [None, 1])
    for chains in (1024, 4096):
        compare("glmm6000", 6000, chains, [None])
    if "--g16000" in sys.argv:
        for chains in (1024, 4096):
            compare("glmm16000", 16000, chains, [None])
