"""DESeq_device with size factors vs the same data with a normalization-factor matrix, alternated in one process after
warm-up, on one GPU, at two shapes:
  C2   50 000 x 100,  ~condition
  C4   50 000 x 1000, 10-level factor
Three runs per round: sizeFactors=s, an nf matrix whose every row is s ("const"), and tximport-like factors from an
avgTxLength-style matrix ("tx").  Medians of wall clock ending in torch.cuda.synchronize(), plus CUDA-event times of
normalization_factors (the tximport estimation) and of the nf prep call (b200nb_prep_nf_dev) next to the size-factor
prep call.  Prints one JSON line with the card name and power limit read in the same run.
usage: python scripts/nf_pipeline.py [reps]"""
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
    n, m = 50000, (100 if name == "C2" else 1000)
    x = synth.design_condition(m) if name == "C2" else synth.design_factor(m, 10)
    d = synth.make_example_counts(n, m, x=x, seed=11)
    sf = d["sizeFactors"]
    y = D.to_gene_major(d["counts"], dev)
    length = np.exp(np.random.default_rng(3).normal(7.0, 0.3, (n, m)))       # average transcript lengths
    txl = D.to_gene_major(length, dev)
    const = D.to_gene_major(np.broadcast_to(sf, (n, m)), dev)
    tx = DP.normalization_factors(y, m, avgTxLength=txl)["normalizationFactors"]
    return {"n": n, "m": m, "x": x, "y": y, "sf": sf, "txl": txl, "nf": {"const": const, "tx": tx}}


def run(s, mode):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if mode == "sf":
        DP.DESeq_device(s["y"], s["x"], s["sf"])
    else:
        DP.DESeq_device(s["y"], s["x"], normalizationFactors=s["nf"][mode])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def events(fn, k):
    ms = []
    for i in range(k + 2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        if i >= 2:
            ms.append(a.elapsed_time(b))
    return ms


out = {"reps": reps}
med = lambda v: round(float(np.median(v)), 2)
modes = ("sf", "const", "tx")
for name in ("C2", "C4"):
    s = shape(name)
    for md in modes:                                               # warm-up
        run(s, md)
    ms = {md: [] for md in modes}
    for _ in range(reps):
        for md in modes:
            ms[md].append(run(s, md))
    est = events(lambda: DP.normalization_factors(s["y"], s["m"], avgTxLength=s["txl"]), reps)
    prep_nf = events(lambda: DP.prep(s["y"], s["x"], None, normalizationFactors=s["nf"]["tx"], xim=1.0), reps)
    prep_sf = events(lambda: DP.prep(s["y"], s["x"], s["sf"]), reps)
    out[name] = {"genes": s["n"], "samples": s["m"], "p": int(s["x"].shape[1]),
                 **{f"{md}_ms_median": med(ms[md]) for md in modes},
                 **{f"{md}_ms": [round(v, 2) for v in ms[md]] for md in modes},
                 "normalization_factors_ms_median": med(est), "prep_nf_call_ms_median": med(prep_nf),
                 "prep_sf_call_ms_median": med(prep_sf)}
    del s
    torch.cuda.empty_cache()

try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:                                              # pragma: no cover
    smi = f"unavailable: {e}"
out["gpu"] = smi
print(json.dumps(out))
