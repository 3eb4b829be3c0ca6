"""BASELINE config 4 as defined (50 000 genes x 1000 samples, 10-level factor, betaPrior=TRUE) on one GPU: DESeq_device
with betaPrior off and on, alternated in one process; the prior-variance kernel alone; per-stage times of one run of
each from B200NB_PIPE_DEBUG=1 (synchronised stage marks, a separate run).  Prints one JSON line.
usage: python scripts/c4_beta_prior.py [reps] [genes]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
n = int(sys.argv[2]) if len(sys.argv) > 2 else 50000
m = 1000
factors = [(np.arange(m) * 10) // m]
x = synth.design_factor(m, 10)
assert np.array_equal(x, pipeline.factorDesign(factors)[0])
d = synth.make_example_counts(n, m, x=x, seed=11)
dev = torch.device("cuda")
y = D.to_gene_major(d["counts"], dev)


def run(prior):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = DP.DESeq_device(y, x, d["sizeFactors"], betaPrior=prior, factors=factors if prior else None)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


for prior in (False, True, False, True):                       # warm-up
    run(prior)
ms = {False: [], True: []}
for _ in range(reps):
    for prior in (False, True):
        ms[prior].append(run(prior)[0])

_, r = run(True)
col_a, col_b, _ = DP.beta_prior_columns(pipeline.factorDesign(factors)[2])
bt = r["mleBetaMatrix"].T.contiguous()
ev = lambda: torch.cuda.Event(enable_timing=True)
kern = []
for i in range(reps + 2):
    a, b = ev(), ev()
    a.record()
    DP.beta_prior_quantile(bt, r["baseMean"], r["dispFit"], col_a, col_b, 0.95)
    b.record()
    torch.cuda.synchronize()
    if i >= 2:
        kern.append(a.elapsed_time(b))

os.environ["B200NB_PIPE_DEBUG"] = "1"
stages = {}
for prior in (False, True):
    stages["on" if prior else "off"] = run(prior)[1]["stage_ms"]
os.environ.pop("B200NB_PIPE_DEBUG")

try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:                                          # pragma: no cover
    smi = f"unavailable: {e}"
med = lambda v: float(np.median(v))
print(json.dumps({"genes": n, "samples": m, "levels": 10, "reps": reps, "gpu": smi,
                  "betaPrior_off_ms_median": round(med(ms[False]), 2), "betaPrior_on_ms_median": round(med(ms[True]), 2),
                  "betaPrior_off_ms": [round(v, 2) for v in ms[False]], "betaPrior_on_ms": [round(v, 2) for v in ms[True]],
                  "prior_var_kernel_ms_median": round(med(kern), 3), "prior_var_columns": len(col_a),
                  "stage_ms": stages, "betaPriorVar": [float(v) for v in r["betaPriorVar"]]}))
