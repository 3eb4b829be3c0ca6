"""DESeq_device + results_device with useT off and on, alternated in one process, on one GPU, at three shapes:
  C2   50 000 x 100,  ~condition
  C4   50 000 x 1000, 10-level factor (p = 11: 550 000 Wald tails)
  sc   20 000 x 2000, ~condition, poscounts size factors, minmu = 1e-6, observation weights with ~30 % of entries near
       zero (non-integer df = rowSums(normalised weights) - p)
and device_pipeline.t_wald_pvalue alone on each shape's (n, p) Wald statistics and df (CUDA events).  Prints one
JSON line with the card name and power limit read in the same run.
usage: python scripts/useT_pipeline.py [reps]"""
import json
import os
import subprocess
import sys
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


def shape(name):
    kw = {}
    if name == "C2":
        n, m, x = 50000, 100, synth.design_condition(100)
    elif name == "C4":
        n, m, x = 50000, 1000, synth.design_factor(1000, 10)
    else:
        n, m, x = 20000, 2000, synth.design_condition(2000)
        kw = {"minmu": 1e-6}
    d = synth.make_example_counts(n, m, x=x, seed=11)
    counts, sf = d["counts"], d["sizeFactors"]
    if name == "sc":
        counts = counts.copy()
        low = np.random.default_rng(3).random(counts.shape) < 0.3
        counts[low] = 0
        w = np.random.default_rng(5).uniform(0.5, 1.0, (n, m))
        w[low] = 10.0 ** np.random.default_rng(6).uniform(-4, -2, int(low.sum()))
        w[:, 0] = 1.0
        y = D.to_gene_major(counts, dev)
        sf = DP.size_factors(y, m, type="poscounts")["sizeFactors"].cpu().numpy()
        kw["weights"] = D.to_gene_major(w, dev)
    else:
        y = D.to_gene_major(counts, dev)
    return {"n": n, "m": m, "x": x, "y": y, "sf": sf, "kw": kw}


def run(s, useT):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = DP.DESeq_device(s["y"], s["x"], s["sf"], useT=useT, **s["kw"])
    DP.results_device(res, s["y"], s["x"], name=1, weights=s["kw"].get("weights"))
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, res


out = {"reps": reps}
med = lambda v: round(float(np.median(v)), 2)
for name in ("C2", "C4", "sc"):
    s = shape(name)
    try:
        for t in (False, True):                                  # warm-up
            run(s, t)
    except FloatingPointError as e:
        out[name] = {"failed": str(e)}
        continue
    ms = {False: [], True: []}
    res = None
    for _ in range(reps):
        for t in (False, True):
            v, r = run(s, t)
            ms[t].append(v)
            if t:
                res = r
    z, df = res["WaldStatistic"].contiguous(), res["tDegreesFreedom"][:, None]
    tail = []
    for i in range(reps + 2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        DP.t_wald_pvalue(z, df)
        b.record()
        torch.cuda.synchronize()
        if i >= 2:
            tail.append(a.elapsed_time(b))
    out[name] = {"genes": s["n"], "samples": s["m"], "p": int(s["x"].shape[1]), "tails": int(z.numel()),
                 "df_min": float(torch.nan_to_num(res["tDegreesFreedom"], nan=np.inf).min()),
                 "useT_off_ms_median": med(ms[False]), "useT_on_ms_median": med(ms[True]),
                 "useT_off_ms": [round(v, 2) for v in ms[False]], "useT_on_ms": [round(v, 2) for v in ms[True]],
                 "t_wald_pvalue_ms_median": med(tail)}
    del s, res
    torch.cuda.empty_cache()

try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:                                          # pragma: no cover
    smi = f"unavailable: {e}"
out["gpu"] = smi
print(json.dumps(out))
