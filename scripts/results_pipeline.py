"""Times results() on the device (results_device and its kernels: b200nb_results_gene_dev, b200nb_filter_cutoffs_dev,
b200nb_filter_numrej_dev, b200nb_padj_dev) after DESeq_device, and prints one JSON line.  Run on the GPU:
    python scripts/results_pipeline.py [--out DIR]
  * DESeq_device and results_device (defaults: last coefficient, Cook's cutoff with the two-group heuristic, BH with
    independent filtering) end to end, host clock ending in a device synchronise, alternated after one warm-up call;
  * each kernel alone: CUDA events around `--kreps` calls after 3 warm-up calls, on the vectors of one results_device
    call (the heuristic kernel on the genes the default Cook's cutoff flags);
  * where results_device's time goes: its stages called one by one, each timed by a host clock ending in a device
    synchronise (the column and per-gene kernel; the flagged-row count and the Cook's rows recomputed for the
    heuristic; the p-value sort, cutoffs and counts up to the numRej read; lowess and the choice of theta on the host;
    the adjusted column);
at C2 (50 000 x 100) and C4 (50 000 x 1000), ~condition counts.  The card name and power limit are read in the same
run."""
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
from scipy import stats                             # noqa: E402


def stages(DP, ds, y, ynz, x, m, cols, cooks_cut, keep, sf, out, reps):
    """Median ms of results_device's stages, each called alone and ended by a device synchronise."""
    from deseq2_b200.pipeline import filter_choose, lowess
    dev = y.device
    sfd = torch.as_tensor(sf, device=dev)
    th = torch.as_tensor(out["metadata"]["filterNumRej"]["theta"], device=dev)
    nr = out["metadata"]["filterNumRej"]

    def heuristic():
        rows = torch.nonzero(ds["maxCooks"] > cooks_cut).squeeze(1)
        DP.results_heuristic(ynz, m, rows, DP._first_fit_cooks(ds, ynz, rows, x, sfd), keep)

    def counts():
        ps, order = torch.sort(out["pvalue"])
        fs = out["baseMean"][order].contiguous()
        c = DP.filter_cutoffs(out["baseMean"], th)
        torch.stack([DP.filter_numrej(ps, fs, c, "BH", 0.1).to(torch.float64), th, c]).cpu()

    def host_lowess():
        filter_choose(nr["numRej"], lowess(nr["theta"], nr["numRej"], f=1.0 / 5.0)["y"])

    ps, order = torch.sort(out["pvalue"])
    fs = out["baseMean"][order].contiguous()
    c = DP.filter_cutoffs(out["baseMean"], th)
    calls = {"column+results_gene": lambda: DP.results_gene(ynz, m, *cols, maxCooks=ds["maxCooks"],
                                                            cooksCutoff=cooks_cut, keep=keep),
             "heuristic (flag count, Cook's rows, kernel)": heuristic,
             "sort+cutoffs+numrej+read": counts,
             "lowess+choice (host)": host_lowess,
             "padj": lambda: DP.padj_column(ps, fs, order, "BH", c, out["metadata"]["j"])}
    for f in calls.values():
        f()
    return {k: float(np.median([timed(f) for _ in range(reps)])) for k, f in calls.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--kreps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    dev = torch.device("cuda")
    res = {"card": card(), "shapes": {}}
    for name, n, m in (("C2", 50000, 100), ("C4", 50000, 1000)):
        factors = [np.repeat([0, 1], m // 2)]
        x = pipeline.factorDesign(factors)[0]
        d = synth.make_example_counts(n, m, x=x, seed=4)
        y = D.to_gene_major(d["counts"].astype(np.int32), dev)
        sf = d["sizeFactors"]
        r = {"n": n, "m": m}
        ds = DP.DESeq_device(y, x, sizeFactors=sf)
        out = DP.results_device(ds, y, x, factors=factors)
        r["filterTheta"] = out["metadata"]["filterTheta"]
        r["rejections"] = int((out["padj"] < 0.1).sum().item())
        runs = {"DESeq_device": [], "results_device": []}
        for _ in range(a.reps):
            runs["DESeq_device"].append(timed(lambda: DP.DESeq_device(y, x, sizeFactors=sf)))
            ds = DP.DESeq_device(y, x, sizeFactors=sf)
            runs["results_device"].append(timed(lambda: DP.results_device(ds, y, x, factors=factors)))
        r["end_to_end_ms"] = {k: float(np.median(v)) for k, v in runs.items()}
        r["end_to_end_ms_all"] = runs
        ynz = y[ds["idx"]].contiguous()
        cols = [ds[k][:, 1].contiguous() for k in ("betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue")]
        cooks_cut = float(stats.f.ppf(0.99, 2, m - 2))
        flagged = torch.nonzero(ds["maxCooks"] > cooks_cut).squeeze(1)
        keep = torch.zeros(ynz.shape[0], dtype=torch.int32, device=dev)
        ck = DP._first_fit_cooks(ds, ynz, flagged, x, torch.as_tensor(sf, device=dev))
        r["flagged"] = int(flagged.numel())
        pv, filt = out["pvalue"], out["baseMean"]
        ps, order = torch.sort(pv)
        fs = filt[order].contiguous()
        th = torch.as_tensor(out["metadata"]["filterNumRej"]["theta"], device=dev)
        cutoffs = DP.filter_cutoffs(filt, th)
        r["kernel_ms"] = {
            "results_gene": event_ms(lambda: DP.results_gene(ynz, m, *cols, maxCooks=ds["maxCooks"],
                                                             cooksCutoff=cooks_cut, keep=keep), a.kreps),
            "results_heuristic": event_ms(lambda: DP.results_heuristic(ynz, m, flagged, ck, keep), a.kreps),
            "filter_cutoffs": event_ms(lambda: DP.filter_cutoffs(filt, th), a.kreps),
            "filter_numrej": event_ms(lambda: DP.filter_numrej(ps, fs, cutoffs, "BH", 0.1), a.kreps),
            "padj": event_ms(lambda: DP.padj_column(ps, fs, order, "BH", cutoffs, out["metadata"]["j"]), a.kreps)}
        r["stage_ms"] = stages(DP, ds, y, ynz, x, m, cols, cooks_cut, keep, sf, out, a.reps)
        res["shapes"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "results_pipeline.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
