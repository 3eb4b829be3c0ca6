"""DESeq_device with observation weights off and on, alternated in one process, on one GPU, at three shapes:
  C2   50 000 x 100,  ~condition
  C4   50 000 x 1000, 10-level factor, betaPrior off
  sc   20 000 x 2000, ~condition, poscounts size factors, minmu = 1e-6, weights with ~30 % of entries near zero
and the weighted prep kernel alone (b200nb_prep_weighted_dev, CUDA events).  Prints one JSON line with the card name
and power limit read in the same run.
usage: python scripts/weights_pipeline.py [reps]"""
import json
import subprocess
import sys
import os
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deseq2_b200 import device as D, device_pipeline as DP, synth  # noqa: E402

warnings.simplefilter("ignore")
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
dev = torch.device("cuda")


def zi_weights(n, m, seed, low=None):
    """most weights in (0.5, 1]; ~30 % near zero (1e-4 .. 1e-2): at `low` (the dropouts) when given"""
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.5, 1.0, (n, m))
    if low is None:
        low = rng.random((n, m)) < 0.3
    w[low] = 10.0 ** rng.uniform(-4, -2, int(low.sum()))
    w[:, 0] = 1.0
    return w


def shape(name):
    if name == "C2":
        n, m, x, kw = 50000, 100, synth.design_condition(100), {}
    elif name == "C4":
        n, m, x, kw = 50000, 1000, synth.design_factor(1000, 10), {}
    else:
        n, m, x, kw = 20000, 2000, synth.design_condition(2000), {"minmu": 1e-6}
    d = synth.make_example_counts(n, m, x=x, seed=11)
    counts = d["counts"]
    sf = d["sizeFactors"]
    low = None
    if name == "sc":                                             # dropouts, which the weights down-weight
        counts = counts.copy()
        low = np.random.default_rng(3).random(counts.shape) < 0.3
        counts[low] = 0
    y = D.to_gene_major(counts, dev)
    if name == "sc":
        sf = DP.size_factors(y, m, type="poscounts")["sizeFactors"].cpu().numpy()
    w = D.to_gene_major(zi_weights(n, m, 5, low), dev)
    return {"n": n, "m": m, "x": x, "y": y, "sf": sf, "w": w, "kw": kw}


def run(s, weighted):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    DP.DESeq_device(s["y"], s["x"], s["sf"], weights=s["w"] if weighted else None, **s["kw"])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


out = {"reps": reps}
med = lambda v: round(float(np.median(v)), 2)
for name in ("C2", "C4", "sc"):
    s = shape(name)
    try:
        for wt in (False, True):                                 # warm-up
            run(s, wt)
    except FloatingPointError as e:                              # e.g. the parametric trend fit failed
        out[name] = {"failed": str(e)}
        continue
    ms = {False: [], True: []}
    for _ in range(reps):
        for wt in (False, True):
            ms[wt].append(run(s, wt))
    ev = lambda: torch.cuda.Event(enable_timing=True)
    kern = []
    for i in range(reps + 2):
        a, b = ev(), ev()
        a.record()
        DP.prep(s["y"], s["x"], s["sf"], want_mu=False, weights=s["w"])
        b.record()
        torch.cuda.synchronize()
        if i >= 2:
            kern.append(a.elapsed_time(b))
    out[name] = {"genes": s["n"], "samples": s["m"], "p": int(s["x"].shape[1]), "weights_off_ms_median": med(ms[False]),
                 "weights_on_ms_median": med(ms[True]), "weights_off_ms": [round(v, 2) for v in ms[False]],
                 "weights_on_ms": [round(v, 2) for v in ms[True]], "weighted_prep_call_ms_median": med(kern)}
    del s
    torch.cuda.empty_cache()

try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:                                          # pragma: no cover
    smi = f"unavailable: {e}"
out["gpu"] = smi
print(json.dumps(out))
