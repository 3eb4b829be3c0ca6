"""Times DESeq(sfType = "iterate") on the device (size_factors_iterate, b200nb_sf_iterate_objective_dev) and prints one
JSON line.  Run on the GPU:  python scripts/sf_iterate.py [--out DIR]
  * objective-call time (CUDA events around b200nb_sf_iterate_objective_dev, 20 calls after 3 warm-up calls) at C2
    (50 000 x 100) and at a single-cell-like 20 000 x 2000 shape;
  * the whole size_factors_iterate (host clock ending in a device synchronise): outer iterations, objective calls;
  * DESeq_device(sfType = "iterate", fitType = "mean") against DESeq_device(sfType = "ratio"), alternated in this
    process after one warm-up run of each;
  * the host mirror's direct evaluation (pipeline.iterateObjective) per objective call at the same shapes, on the CPU.
The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                   # pragma: no cover
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    dev = torch.device("cuda")
    res = {"card": card(), "shapes": {}}
    for name, n, m in (("C2", 50000, 100), ("single_cell", 20000, 2000)):
        x = synth.design_condition(m)
        d = synth.make_example_counts(n, m, x=x, seed=17)
        y = D.to_gene_major(d["counts"].astype(np.int32), dev)
        r = {"n": n, "m": m}
        # objective calls at the first iteration's q / dispersions
        keep = d["counts"].sum(axis=1) > 0
        ynz = y[torch.as_tensor(np.flatnonzero(keep), device=dev)].contiguous()
        q, disp, *_ = DP._dispersions_intercept_mean(ynz, m, np.ones(m))
        par = torch.zeros(m, dtype=torch.float64, device=dev)
        out = torch.empty(2 * m + 1, dtype=torch.float64, device=dev)
        for _ in range(3):
            DP.sf_iterate_objective(ynz, q, disp, par, m, out=out)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            DP.sf_iterate_objective(ynz, q, disp, par, m, out=out)
        e1.record()
        torch.cuda.synchronize()
        r["objective_call_ms"] = e0.elapsed_time(e1) / 20
        # host mirror, one direct evaluation of the 2m + 1 columns (C2) or of 5 columns scaled to 2m + 1
        K = d["counts"][keep].astype(np.float64)
        qh, dh = q[:, :m].cpu().numpy(), disp.cpu().numpy()
        cols = 2 * m + 1 if m <= 100 else 5
        t = time.perf_counter()
        p0 = np.zeros(m)
        for c in range(cols):
            p = p0.copy()
            if c > 0:
                p[(c - 1) % m] += 1e-3 if c <= m else -1e-3
            ll = pipeline.nbinomLogLike(K, qh * np.exp(p - p.mean())[None, :], dh)
            ll[ll > np.quantile(ll, 0.05, method="linear")].sum()
        r["host_objective_call_ms"] = (time.perf_counter() - t) * 1e3 * (2 * m + 1) / cols
        r["host_objective_columns_timed"] = cols
        # whole size_factors_iterate
        torch.cuda.synchronize()
        t = time.perf_counter()
        it = DP.size_factors_iterate(y, m)
        torch.cuda.synchronize()
        r["size_factors_iterate_ms"] = (time.perf_counter() - t) * 1e3
        r["outer_iterations"] = it["iterations"]
        r["objective_calls_per_iteration"] = it["evaluations"]
        # DESeq_device iterate vs ratio, alternated
        runs = {"iterate": [], "ratio": []}
        kinds = [("iterate", dict(sfType="iterate", fitType="mean")), ("ratio", dict())]
        for k, kw in kinds:                                                  # warm-up
            DP.DESeq_device(y, x, **kw)
        for _ in range(a.reps):
            for k, kw in kinds:
                torch.cuda.synchronize()
                t = time.perf_counter()
                DP.DESeq_device(y, x, **kw)
                torch.cuda.synchronize()
                runs[k].append((time.perf_counter() - t) * 1e3)
        r["DESeq_device_ms"] = {k: float(np.median(v)) for k, v in runs.items()}
        r["DESeq_device_ms_all"] = runs
        res["shapes"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "sf_iterate.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
