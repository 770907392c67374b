"""
Posterior-predictive draws on the device (rn_generator_*, rn_sample_generate): two workloads.

  eight-schools replicate: traverse(Normal(theta_i, sigma_i)) over 8 192 chains x 1 000 draws (DefaultConfig sampling)
      - device draws per second of rn_generator_eval_device over device-resident draws: host clock around blocking calls
        (each call also copies the chains' RNG states in and out; device buffers are kept by the handle), warm module
      - wall time of sample_generate against sample_predict followed by the host Generator.predict loop.  No JVM exists here:
        the host loop is the Python oracle's closures (labelled as such), timed on --host-chains chains and scaled linearly.
  Poisson-regression replicate: Poisson(exp(a + b x_i)) for 1 000 fixed covariates x_i, at 1 024 / 8 192 / 65 536 chains x
      --poisson-iterations posterior draws (a, b) drawn here: device draws per second, and end to end rn_generator_eval
      from host buffers (draws in, predictive draws out).
Every generator's NVRTC compile (create + first load, `compile_seconds`) is reported and added to the end-to-end figures:
the plan is straight-line code, so it grows with the number of draws per iteration.

Also prints registers / spills of rn_k_generate from `nvcc -Xptxas -v` for both generators, and the card's name and power
limit.  One JSON line per measurement; nothing is written to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.rainier_py import configs  # noqa: E402
from oracle.rainier_py.binding import ScalaRNG  # noqa: E402
from oracle.rainier_py.compute import Real  # noqa: E402
from oracle.rainier_py.core import Model, Normal, Poisson, to_generator  # noqa: E402
from rainier_b200 import api  # noqa: E402
from rainier_b200 import generate as G  # noqa: E402


def ptxas(src):
    with tempfile.TemporaryDirectory() as d:
        cu = os.path.join(d, "g.cu")
        with open(cu, "w") as f:
            f.write(src)
        r = subprocess.run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17",
                            "--fmad=false", "-cubin", "-Xptxas", "-v", "-o", os.path.join(d, "g.cubin"), cu], capture_output=True, text=True)
    lines = (r.stdout + r.stderr).splitlines()
    out, cur = {}, None
    for ln in lines:
        if "Compiling entry function" in ln:
            cur = ln.split("'")[1]
        elif cur and "Used" in ln and "registers" in ln:
            out[cur] = {"registers": int(ln.split("Used")[1].split("registers")[0]), "line": ln.strip()}
        elif cur and "spill" in ln:
            out.setdefault(cur, {})["spill"] = ln.strip()
    return out.get("rn_k_generate", {"error": r.returncode})


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return {"card": name, "power_limit": pl}


def device_rate(g, chains, iters, n, reps, x_fn):
    """rn_generator_eval_device over device-resident sampler-layout draws; host clock around `reps` blocking calls"""
    import torch
    dev = torch.device("cuda:0")
    d_x = torch.from_numpy(np.ascontiguousarray(x_fn())).to(dev)  # [iterations][n][chains]
    d_out = torch.empty((chains, iters, g.nOutputs), dtype=torch.float64, device=dev)
    states = [ScalaRNG(1000 + c).rand.state() for c in range(chains)]
    states = g.eval_device(d_x.data_ptr(), iters, chains, states, d_out.data_ptr())  # warm: module load, allocations
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        states = g.eval_device(d_x.data_ptr(), iters, chains, states, d_out.data_ptr())
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / reps
    return {"seconds_per_call": dt, "draws": chains * iters * g.nOutputs, "draws_per_second": chains * iters * g.nOutputs / dt}


def eight_schools(a, info):
    model, mu, tau, thetas, sigmas = configs.eight_schools_parts()
    rir, cols = model.compile(True)
    t = [Normal(thetas.at(i), sigmas[i]) for i in range(8)]
    grir = G.lower_generator(t, model.parameters)
    g, t_compile = compiled(grir)
    C, I = a.chains, a.iterations
    rng = np.random.default_rng(0)
    r = device_rate(g, C, I, 10, a.reps, lambda: rng.normal(size=(I, 10, C)))
    print(json.dumps(dict(info, workload="eight_schools_replicate", chains=C, iterations=I, metric="device_generate", **r)))
    m = api.CudaModel(rir, cols)
    config = api.SamplerConfig(iterations=I)
    seeds = np.arange(C, dtype=np.int64) + 1
    m.sample_generate(g, api.SamplerConfig(iterations=10, warmupIterations=10), seeds=seeds[:64])  # warm kernels
    t0 = time.perf_counter()
    m.sample_generate(g, config, seeds=seeds)
    t_gen = time.perf_counter() - t0
    f = api.CudaFunction(compile_reqs(t, model.parameters))
    t0 = time.perf_counter()
    pred, tr = m.sample_predict(f, config, seeds=seeds)
    t_pred = time.perf_counter() - t0
    # host loop of the Python oracle over --host-chains chains (the reference's per-draw Generator.get), scaled to C chains
    gen = to_generator(t)
    reqs = gen.reqs()
    from oracle.rainier_py.compute import Evaluator
    t0 = time.perf_counter()
    for c in range(a.host_chains):
        rr = ScalaRNG(int(seeds[c]))
        for row in pred[c]:
            cache = dict(zip(reqs, (float(v) for v in row)))
            gen.get(rr, Evaluator(cache))
    t_host = (time.perf_counter() - t0) * C / a.host_chains
    print(json.dumps(dict(info, workload="eight_schools_replicate", chains=C, iterations=I, metric="end_to_end_seconds",
                          compile_seconds=t_compile, sample_generate=t_gen, sample_generate_plus_compile=t_gen + t_compile,
                          sample_predict=t_pred,
                          host_predict_loop_python_oracle_scaled=t_host, host_loop_measured_chains=a.host_chains,
                          sample_predict_plus_host_loop=t_pred + t_host)))
    return g


def compiled(rir):
    """a CudaGenerator with its module compiled and loaded, and the seconds that took"""
    t0 = time.perf_counter()
    g = api.CudaGenerator(rir)
    g.emit_cubin()
    return g, time.perf_counter() - t0


def compile_reqs(t, params):
    from oracle.rainier_py.compute import compile_function_rir
    return compile_function_rir(params, to_generator(t).reqs())


def poisson_regression(a, info):
    xs = np.random.default_rng(7).normal(size=1000)
    holder = {}

    def keep(v):
        holder["t"] = list(v)
        return Real.sum(list(v))

    Real.parameters(2, keep)
    params = Model.track_(list(holder["t"])).parameters
    qa, qb = holder["t"]
    t = [Poisson((qa + qb * float(x)).exp()) for x in xs]
    g, t_compile = compiled(G.lower_generator(t, params))
    for C in (1024, 8192, 65536):
        I = a.poisson_iterations
        rng = np.random.default_rng(C)
        ab = np.stack([rng.normal(1.0, 0.1, size=(I, C)), rng.normal(0.3, 0.05, size=(I, C))], axis=1)  # [iteration][2][chain]
        r = device_rate(g, C, I, 2, max(1, a.reps // 2), lambda: ab)
        e2e = {"end_to_end_host_buffers": "not measured (%.0f GB of output)" % (C * I * g.nOutputs * 8 / 1e9)}
        if C * I * g.nOutputs * 8 <= 8e9:
            x = np.ascontiguousarray(ab.transpose(2, 0, 1))  # [chain][iteration][2]
            states = [ScalaRNG(1000 + c).rand.state() for c in range(C)]
            t0 = time.perf_counter()
            g(x, states)
            t_e2e = time.perf_counter() - t0
            e2e = {"end_to_end_host_buffers": t_e2e, "end_to_end_plus_compile": t_e2e + t_compile}
        print(json.dumps(dict(info, workload="poisson_regression_replicate_1000", chains=C, iterations=I, metric="device_generate",
                              compile_seconds=t_compile, **e2e, **r)), flush=True)
    return g


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--chains", type=int, default=8192)
    p.add_argument("--iterations", type=int, default=1000)
    p.add_argument("--poisson-iterations", type=int, default=100)
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--host-chains", type=int, default=4)
    a = p.parse_args()
    info = card()
    g1 = eight_schools(a, info)
    g2 = poisson_regression(a, info)
    for name, g in (("eight_schools_replicate", g1), ("poisson_regression_replicate_1000", g2)):
        print(json.dumps(dict(info, workload=name, metric="rn_k_generate_ptxas", **ptxas(g.emit_source()))), flush=True)


if __name__ == "__main__":
    main()
