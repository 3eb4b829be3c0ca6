"""Times DESeq(test = "LRT") on the device, and checks in the same run that the one-call path agrees with the two-call
sequence.  Run on the GPU:
    python scripts/lrt_pipeline.py [--out DIR] [--reps 5] [--scale 1.0]
Three runs per shape, in one process on one GPU, alternated after one warm-up call each; each time is a host clock
ending in a device synchronise, and the median is reported:
  * "wald": DESeq_device (the Wald test);
  * "wald+nbinomLRT": DESeq_device followed by nbinomLRT_device on its dispersions (what bench.py's C5 times);
  * "lrt": DESeq_device(test="LRT", reduced=...), which reuses the Wald fit as the LRT's full fit.
Shapes:
  * C5 at one GPU's share of eight: 125 000 x 200, ~batch + condition vs ~batch;
  * C2: 50 000 x 100, ~condition vs ~1 (DESeq_device(test="LRT") takes R's closed form for ~1, nbinomLRT_device an
    IRLS fit, so there only the full-model columns are compared);
  * single-cell-like: 20 000 x 2000, poscounts size factors, minmu = 1e-6, ~condition vs ~1.
Agreement: the columns the sequence and the one-call path share (bit for bit: betaMatrix, betaSE, deviance and, for a
reduced design other than ~1, LRTStatistic / LRTPvalue; with ~1 the largest relative LRTStatistic difference is
reported).  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from rlog_pipeline import card, timed    # noqa: E402


def shapes(scale):
    from deseq2_b200 import synth
    x5 = synth.design_batch_condition(200, 2)
    x2 = synth.design_condition(100)
    xs = synth.design_condition(2000)
    return [("C5_shard_of_8", int(125000 * scale), 200, x5, x5[:, :2], {}),
            ("C2", int(50000 * scale), 100, x2, np.ones((100, 1)), {}),
            ("single_cell", int(20000 * scale), 2000, xs, np.ones((2000, 1)), {"poscounts": True, "minmu": 1e-6})]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from deseq2_b200 import device as D, device_pipeline as DP, synth
    dev = torch.device("cuda")
    res = {"card (name, power limit)": card(), "shapes": {}}
    for name, n, m, x, xr, opt in shapes(a.scale):
        d = synth.make_example_counts(n, m, x=x, seed=5)
        K = d["counts"]
        if opt.get("poscounts"):
            K = np.where(np.random.default_rng(3).random(K.shape) < 0.3, 0, K)    # dropouts
        y = D.to_gene_major(K.astype(np.int32), dev)
        if opt.get("poscounts"):
            sf = DP.size_factors(y, m, type="poscounts")["sizeFactors"]
            sf = (sf / torch.exp(torch.log(sf).mean())).cpu().numpy()
        else:
            sf = d["sizeFactors"]
        kw = {"minmu": opt.get("minmu", 0.5)}

        def wald():
            return DP.DESeq_device(y, x, sf, **kw)

        def sequence():
            r = DP.DESeq_device(y, x, sf, **kw)
            ynz = y[r["idx"]].contiguous()
            return r, DP.nbinomLRT_device(ynz, x, xr, sf, r["dispersion"], minmu=kw["minmu"])

        def lrt():
            return DP.DESeq_device(y, x, sf, test="LRT", reduced=xr, **kw)

        runs = {"wald": wald, "wald+nbinomLRT": sequence, "lrt": lrt}
        for f in runs.values():
            f()
        times = {k: [] for k in runs}
        for _ in range(a.reps):
            for k, f in runs.items():
                times[k].append(timed(f))
        r = {"n": n, "m": m, "p": x.shape[1], "p_reduced": xr.shape[1], **opt,
             "ms": {k: float(np.median(v)) for k, v in times.items()}, "ms_all": times}
        one = lrt()
        one = {k: v.clone() if isinstance(v, torch.Tensor) else v for k, v in one.items()}
        _, seq = sequence()
        same = lambda k: bool(torch.equal(torch.nan_to_num(one[k], nan=-7.0), torch.nan_to_num(seq[k], nan=-7.0)))
        keys = ["betaMatrix", "betaSE", "deviance"]
        if xr.shape[1] > 1 or not np.all(xr == 1):
            keys += ["LRTStatistic", "LRTPvalue"]
        else:
            s1, s2 = one["LRTStatistic"], seq["LRTStatistic"]
            r["lrt_stat_closed_form_vs_irls_max_abs_diff_over_1_plus_dev"] = float(
                ((s1 - s2).abs() / (1 + one["deviance"].abs())).max().item())
        r["bit_identical"] = {k: same(k) for k in keys}
        r["n_genes"] = int(one["idx"].numel())
        res["shapes"][name] = r
        print(name, json.dumps({k: v for k, v in r.items() if k != "ms_all"}), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "lrt_pipeline.json"), "w") as f:
            f.write(line + "\n")
    assert all(all(r["bit_identical"].values()) for r in res["shapes"].values()), "the two paths disagree"


if __name__ == "__main__":
    main()
