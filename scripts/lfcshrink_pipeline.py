"""Times lfcShrink(type = "normal") on the device (lfcShrink_device: the prior-variance kernel
b200nb_beta_prior_quantile_dev and the MAP fit's IRLS / log-likelihood / optim kernels) after DESeq_device and
results_device, and prints one JSON line.  Run on the GPU:
    python scripts/lfcshrink_pipeline.py [--out DIR]
  * DESeq_device + results_device against the same + lfcShrink_device (given results_device's table), end to end,
    host clock ending in a device synchronise, alternated after one warm-up call, median of --reps calls; and
    lfcShrink_device alone;
  * the prior-variance launch and the MAP fit (_map_fit: IRLS, log-likelihood, optim fallback) alone, CUDA events
    around --kreps calls after 3 warm-up calls;
at C2 (50 000 x 100, ~condition, coef) and C4 (50 000 x 1000, a 10-level factor, a level contrast shrunk on the
expanded matrix, p = 11).  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from rlog_pipeline import card, event_ms, timed    # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--kreps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    dev = torch.device("cuda")
    res = {"card": card(), "shapes": {}}
    for name, n, m, levels, sel in (("C2", 50000, 100, 2, dict(coef=1)),
                                    ("C4", 50000, 1000, 10, dict(contrast=(0, 2, 1)))):
        factors = [(np.arange(m) * levels) // m]
        x = pipeline.factorDesign(factors)[0]
        d = synth.make_example_counts(n, m, x=x, seed=4)
        y = D.to_gene_major(d["counts"].astype(np.int32), dev)
        sf = d["sizeFactors"]
        rsel = dict(name=sel["coef"]) if "coef" in sel else sel
        r = {"n": n, "m": m, "selection": {k: list(v) if isinstance(v, tuple) else v for k, v in sel.items()}}

        def base():
            ds = DP.DESeq_device(y, x, sizeFactors=sf)
            return ds, DP.results_device(ds, y, x, factors=factors, **rsel)

        def shrunk():
            ds, tab = base()
            return DP.lfcShrink_device(ds, y, x, factors=factors, results=tab, **sel)

        out = shrunk()                                              # warm-up
        r["betaPriorVar"] = out["metadata"]["priorInfo"]["betaPriorVar"].tolist()
        r["n_optim"] = out["shrinkFit"]["n_optim"]
        r["map_unconverged"] = int((~out["shrinkFit"]["betaConv"]).sum().item())
        runs = {"DESeq+results": [], "DESeq+results+lfcShrink": [], "lfcShrink_device": []}
        for _ in range(a.reps):
            runs["DESeq+results"].append(timed(base))
            runs["DESeq+results+lfcShrink"].append(timed(shrunk))
            ds, tab = base()
            runs["lfcShrink_device"].append(timed(lambda: DP.lfcShrink_device(ds, y, x, factors=factors, results=tab,
                                                                              **sel)))
        r["end_to_end_ms"] = {k: float(np.median(v)) for k, v in runs.items()}
        r["end_to_end_ms_all"] = runs
        # ---- the two hot stages alone, on the inputs of the last call
        expanded = "contrast" in sel
        p = x.shape[1]
        B, bm, dfit = ds["betaMatrix"], ds["baseMean"], ds["dispFit"]
        if expanded:
            col_a, col_b, _ = DP.beta_prior_columns(pipeline.factorDesign(factors)[2])
        else:
            col_a, col_b = np.arange(1, p, dtype=np.int32), np.full(p - 1, -1, np.int32)
        bt = B.T.contiguous()
        pv = DP.estimate_beta_prior_var(B, factors, bm, dfit, expandedType=expanded)
        ynz = y[ds["idx"]].contiguous()
        sfd = torch.as_tensor(sf, device=dev)
        if expanded:
            xf = pipeline.factorDesign(factors, expanded=True)[0]
            beta0 = DP._expanded_start(bm, xf.shape[1])
        else:
            xf = x
            beta0 = DP.prep(ynz, x, sf, want_mu=False, xim=1.0)["beta0"]
        r["columns"] = int(len(col_a))
        r["kernel_ms"] = {
            "beta_prior_quantile": event_ms(lambda: DP.beta_prior_quantile(bt, bm, dfit, col_a, col_b, 0.95), a.kreps),
            "estimate_beta_prior_var": event_ms(lambda: DP.estimate_beta_prior_var(B, factors, bm, dfit,
                                                                                   expandedType=expanded), a.kreps),
            "map_fit": event_ms(lambda: DP._map_fit(ynz, xf, sfd, ds["dispersion"], pv, beta0, 1e-8, 100, 0.5, True),
                                a.kreps)}
        res["shapes"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "lfcshrink_pipeline.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
