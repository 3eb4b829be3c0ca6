"""Times rlog on the device (rlog_device and its two kernels, b200nb_rlog_fit_dev and b200nb_rlog_prior_var_dev)
next to the VST, and prints one JSON line.  Run on the GPU:  python scripts/rlog_pipeline.py [--out DIR]
  * the fit kernel alone and the prior-variance kernel alone (CUDA events around `--kreps` calls after 3 warm-up
    calls), with the dispFit and betaPriorVar of one rlog_device call;
  * rlog_device (blind), vst_device (nsub = 1000) and varianceStabilizingTransformation_device (blind) end to end (host
    clock ending in a device synchronise), alternated after one warm-up call of each;
  * the reference's own fitBeta (oracle/_ref, src/DESeq2.cpp compiled unchanged, one CPU thread, QR branch) on a fixed
    subset of genes with the same design [1 | I_m], lambdas, dispFit and start values, scaled by n / subset: an
    EXTRAPOLATED per-dataset CPU time of rlogData's fit, not a measured one (reported as such).  Not at C4 unless
    --c4-reference is given: there one gene's fit (a QR of a 2001 x 1001 matrix per IRLS step) takes minutes;
at 50 000 x 8, C2 (50 000 x 100) and C4 (50 000 x 1000), ~condition counts.  The card name and power limit are read in
the same run."""
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
LN2 = float(np.log(2.0))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                   # pragma: no cover
        return f"unknown ({e})"


def timed(f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def event_ms(f, reps):
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def reference_fit_s(K, sf, disp, bpv, genes):
    """Seconds of the reference's fitBeta for rlogData's fit of `genes` rows (one thread)."""
    from oracle import ref as R
    m = K.shape[1]
    Kg = K[genes].astype(np.float64)
    x = np.c_[np.ones(m), np.eye(m)]
    lam = np.r_[1e-6, np.full(m, 1.0 / bpv)] / LN2 ** 2
    beta0 = np.zeros((len(genes), m + 1))
    beta0[:, 0] = np.log((Kg / sf).mean(axis=1))
    nf = np.broadcast_to(sf, Kg.shape).copy()
    t = time.perf_counter()
    R.fitBeta(Kg, x, nf, disp[genes], np.r_[1.0, np.zeros(m)], beta0, lam, None, False, 1e-4, 100, True, 0.5)
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--kreps", type=int, default=20)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--c4-reference", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from deseq2_b200 import device as D, device_pipeline as DP, synth
    dev = torch.device("cuda")
    res = {"card": card(), "shapes": {}}
    for name, n, m, ref_genes in (("50000x8", 50000, 8, 2000), ("C2", 50000, 100, 100), ("C4", 50000, 1000, 1 if a.c4_reference else 0)):
        d = synth.make_example_counts(n, m, x=synth.design_condition(m), seed=4)
        K = d["counts"].astype(np.int32)
        y = D.to_gene_major(K, dev)
        r = {"n": n, "m": m}
        rl = DP.rlog_device(y, m)
        sfd = torch.as_tensor(rl["sizeFactors"], device=dev)
        disp, bpv = rl["dispFit"], rl["betaPriorVar"]
        bm = (y[:, :m].to(torch.float64) / sfd).mean(dim=1)
        it = rl["betaIter"][torch.as_tensor(K.sum(axis=1) > 0, device=dev)]
        r["betaPriorVar"] = bpv
        r["betaIter_mean"] = float(it.mean().item())
        r["betaIter_max"] = float(it.max().item())
        r["kernel_ms"] = {"rlog_fit": event_ms(lambda: DP.rlog_fit(y, m, sfd, disp, bpv), a.kreps),
                          "rlog_prior_var": event_ms(lambda: DP.rlog_prior_var(y, m, sfd, bm, disp), a.kreps)}
        calls = {"rlog_device": lambda: DP.rlog_device(y, m),
                 "vst_device": lambda: DP.vst_device(y, m),
                 "varianceStabilizingTransformation_device": lambda: DP.varianceStabilizingTransformation_device(y, m)}
        for f in calls.values():                                              # warm-up
            f()
        runs = {k: [] for k in calls}
        for _ in range(a.reps):
            for k, f in calls.items():
                runs[k].append(timed(f))
        r["end_to_end_ms"] = {k: float(np.median(v)) for k, v in runs.items()}
        r["end_to_end_ms_all"] = runs
        if not a.no_reference and ref_genes:
            genes = np.flatnonzero(K.sum(axis=1) > 0)[:ref_genes]
            s = reference_fit_s(K, rl["sizeFactors"], disp.cpu().numpy(), bpv, genes)
            r["reference_fit"] = {"genes_timed": int(len(genes)), "measured_s": s,
                                  "extrapolated_dataset_s": s * n / len(genes),
                                  "note": "extrapolated from the timed subset, one CPU thread; not a measured "
                                          "per-dataset time"}
        res["shapes"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "rlog_pipeline.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
