"""results() on the device (device_pipeline.results_device: csrc/results.cuh through the C ABI) against the host mirror
pipeline.results, which restates R/results.R literally (the full filtered_p matrix, p.adjust, quantile type 7, lowess);
the host pieces against scipy, hand-worked vectors and an independent local-linear fit; the selection rules and the
expectations of the reference's tests/testthat/test_results.R that have a Python equivalent.  The CPU tests run the
engine's CUDA source on the SIMT emulator (`emu` fixture); the `-m gpu` tests run on a GPU, or on the emulator when
B200NB_LIB points at it."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm
from deseq2_b200 import pipeline, synth
from ranks import DEVICE, nccl_world, run_ranks

NAN = np.nan


# ---------------------------------------------------------------- host pieces

def test_p_adjust_bh_by_against_scipy():
    from scipy import stats
    rng = np.random.default_rng(1)
    p = rng.uniform(0, 1, 500) ** 3
    p[::17] = p[3]                                            # ties
    for method, sm in (("BH", "bh"), ("fdr", "bh"), ("BY", "by")):
        assert np.allclose(pipeline.p_adjust(p, method), stats.false_discovery_control(p, method=sm), rtol=1e-13)
    q = p.copy()
    q[[4, 9]] = NAN                                           # n counts the non-NA p-values only
    got = pipeline.p_adjust(q, "BH")
    assert np.all(np.isnan(got[[4, 9]]))
    keep = ~np.isnan(q)
    assert np.allclose(got[keep], stats.false_discovery_control(q[keep], method="bh"), rtol=1e-13)


def test_p_adjust_hand_worked():
    p = np.array([0.01, NAN, 0.04, 0.03, 0.03, 0.5])             # n = 5
    assert np.allclose(pipeline.p_adjust(p, "bonferroni"), [0.05, NAN, 0.2, 0.15, 0.15, 1.0], equal_nan=True)
    # holm: sorted 0.01 0.03 0.03 0.04 0.5 -> 5p, 4p, 3p, 2p, 1p = .05 .12 .09 .08 .5 -> cummax .05 .12 .12 .12 .5
    assert np.allclose(pipeline.p_adjust(p, "holm"), [0.05, NAN, 0.12, 0.12, 0.12, 0.5], equal_nan=True)
    # hochberg: (n + 1 - r) p = .05 .12 .09 .08 .5 -> cummin from the top .05 .08 .08 .08 .5
    assert np.allclose(pipeline.p_adjust(p, "hochberg"), [0.05, NAN, 0.08, 0.08, 0.08, 0.5], equal_nan=True)
    assert np.array_equal(pipeline.p_adjust(p, "none"), p, equal_nan=True)
    assert np.array_equal(pipeline.p_adjust([0.3, NAN], "BH"), [0.3, NAN], equal_nan=True)   # n <= 1: p unchanged
    with pytest.raises(ValueError, match="hommel"):
        pipeline.p_adjust(p, "hommel")


def _loclin(x, y, xs, ns, rw):
    """Independent local-linear fit: the ns nearest x (ties at the radius included), tricube weights of distance over
    the radius times rw, weighted least squares through numpy's lstsq."""
    d = np.abs(x - xs)
    h = np.sort(d)[ns - 1]
    u = np.where(d <= 0.999 * h, np.where(d <= 0.001 * h, 1.0, (1 - (d / max(h, 1e-300)) ** 3) ** 3), 0.0) * rw
    sw = np.sqrt(u)
    A = np.c_[np.ones_like(x), x - xs] * sw[:, None]
    return np.linalg.lstsq(A, y * sw, rcond=None)[0][0]


def _brute_lowess(x, y, f, iters):
    n = len(x)
    ns = max(2, min(n, int(f * n + 1e-7)))
    rw = np.ones(n)
    for it in range(iters + 1):
        fit = np.array([_loclin(x, y, xs, ns, rw) for xs in x])
        if it == iters:
            return fit
        r = np.abs(y - fit)
        cmad = 6 * np.median(r)
        rw = np.where(r <= 0.001 * cmad, 1.0, np.where(r <= 0.999 * cmad, (1 - (r / cmad) ** 2) ** 2, 0.0))


def test_lowess():
    xi = np.arange(1.0, 51.0)
    assert np.allclose(pipeline.lowess(xi, 3 * xi + 2, f=0.2, iter=0)["y"], 3 * xi + 2, rtol=1e-13)   # a line
    x = np.linspace(0.1, 0.95, 50)
    rng = np.random.default_rng(4)
    y = 5 * x + rng.normal(0, 0.3, 50)
    y[20] += 4.0                                              # one outlier: the robustness passes down-weight it
    plain, robust = (pipeline.lowess(x, y, f=0.3, iter=k)["y"] for k in (0, 3))
    assert abs(plain[20] - 5 * x[20]) > 0.4 and abs(robust[20] - 5 * x[20]) < 0.1
    numRej = np.round(200 * (1 - np.exp(-10 * x)) + rng.normal(0, 5, 50))
    for iters in (0, 3):                                      # the theta grid: delta = 0.01 range skips no point
        got = pipeline.lowess(x, numRej, f=0.2, iter=iters)["y"]
        assert np.allclose(got, _brute_lowess(x, numRej, 0.2, iters), rtol=1e-9, atol=1e-9)
    xr = np.sort(rng.uniform(0, 1, 40))
    yr = np.sin(6 * xr) + rng.normal(0, 0.2, 40)
    got = pipeline.lowess(xr, yr, f=0.4, delta=0.0)["y"]
    assert np.allclose(got, _brute_lowess(xr, yr, 0.4, 3), rtol=1e-9, atol=1e-9)


def test_quantile7():
    x = np.array([3.0, 1.0, 1.0, 1.0, 7.0, 2.0])
    s = np.sort(x)
    probs = np.array([0.0, 0.1, 0.3, 0.5, 0.77, 1.0])
    want = []
    for pr in probs:
        index = 1 + 5 * pr
        lo, hi = int(np.floor(index)), int(np.ceil(index))
        q = s[lo - 1]
        if index > lo and s[hi - 1] != q:
            h = index - lo
            q = (1 - h) * q + h * s[hi - 1]
        want.append(q)
    assert np.array_equal(pipeline.quantile7(x, probs), want)
    assert pipeline.quantile7(x, [0.1])[0] == 1.0             # ties: x[hi] == x[lo], no interpolation
    assert pipeline.quantile7([4.0], [0.0, 1.0]).tolist() == [4.0, 4.0]


def test_default_theta():
    f = np.r_[np.zeros(30), np.arange(1.0, 71.0)]
    th = pipeline.filter_default_theta(f)
    assert th[0] == 0.3 and th[-1] == 0.95 and len(th) == 50
    assert th[7] == 0.3 + 7 * ((0.95 - 0.3) / 49)
    assert np.all(pipeline.filter_default_theta(np.r_[np.zeros(96), 1, 2, 3, 4]) >= 0.96)
    assert pipeline.filter_default_theta(np.r_[np.zeros(96), 1, 2, 3, 4])[-1] == 1.0


def test_selection_rules():
    factors = [np.repeat([0, 1], 6), np.repeat([0, 1, 2], 4)]
    x, names, _, _ = pipeline.factorDesign(factors)
    S = lambda **kw: pipeline.resultsSelection(x, factors=factors, **kw)
    assert S() == {"kind": "coef", "col": 3, "negate": False, "mask": None}
    assert S(name=1)["col"] == 1 and S(name="f12")["col"] == 3
    a = S(contrast=(1, 2, 0))
    assert a["kind"] == "coef" and a["col"] == 3 and not a["negate"] and a["mask"].sum() == 8
    b = S(contrast=(1, 0, 1))
    assert b["kind"] == "coef" and b["col"] == 2 and b["negate"]
    c = S(contrast=(1, 1, 2))
    assert c["kind"] == "contrast" and c["vec"].tolist() == [0, 0, 1, -1] and c["mask"].tolist() == [False] * 4 + [True] * 8
    d = S(contrast=[["f12"], ["f11"]], listValues=(0.5, -0.5))
    assert d["vec"].tolist() == [0, 0, -0.5, 0.5] and d["mask"] is not None
    e = S(contrast=[["f12"]])
    assert e["vec"].tolist() == [0, 0, 0, 1] and e["mask"] is None
    assert S(contrast=np.array([0, 1.0, 0, 0]))["mask"] is None
    xe = pipeline.factorDesign(factors, expanded=True)[0]
    g = pipeline.resultsSelection(x, factors=factors, betaPrior=True, modelMatrix=xe)
    assert g["kind"] == "contrast" and g["vec"].tolist() == [0, 0, 0, -1, 0, 1]     # last factor, last level vs first
    for bad in (dict(name=[1, 2]), dict(name="foo"), dict(contrast=(5, 1, 0)), dict(contrast=(1, 3, 0)),
                dict(contrast=(1, 1, 1)), dict(contrast=False), dict(contrast=("a", "b", "c", "d")),
                dict(contrast=[["f11"], ["f12"], ["f12"]]), dict(contrast=[["f11"], [1]]),
                dict(contrast=[["f11"], ["foo"]]), dict(contrast=[["f11"], ["f11"]]), dict(contrast=[[], []]),
                dict(contrast=np.zeros(6)), dict(contrast=np.zeros(4)), dict(listValues=(1, 1))):
        with pytest.raises(ValueError):
            S(**bad)


def test_results_checks():
    with pytest.raises(ValueError, match="lessAbs"):
        pipeline.results_checks(0, "lessAbs", False, False, 0.1)
    with pytest.raises(ValueError, match="Wald"):
        pipeline.results_checks(1, "greater", True, False, 0.1)
    with pytest.raises(ValueError, match="betaPrior"):
        pipeline.results_checks(1, "lessAbs", False, True, 0.1)
    with pytest.raises(ValueError, match="alpha"):
        pipeline.results_checks(0, "greaterAbs", False, False, 1.0)
    with pytest.raises(ValueError, match="lfcThreshold"):
        pipeline.results_checks(-1, "greaterAbs", False, False, 0.1)
    with pytest.raises(ValueError, match="useT"):
        pipeline.results_checks(0, "greaterAbs", False, False, 0.1, useT=True)
    with pytest.raises(ValueError, match="theta"):
        pipeline.check_filter_args(3, None, [0.5], 0.1, "BH")
    with pytest.raises(ValueError, match="filter function"):
        pipeline.check_filter_args(3, np.mean, None, 0.1, "BH")
    with pytest.raises(ValueError, match="hommel"):
        pipeline.check_filter_args(3, None, None, 0.1, "hommel")


# ---------------------------------------------------------------- device vs host

def _host_inputs(res, y, K, x, dev, nf=None, weights=None):
    """pipeline.DESeq's layout (all N rows) from a DESeq_device result, and the first fit's Cook's matrix; weights: the
    raw weights (numpy), whose weightsFail rows keep pipeline.DESeq's weighted baseMean."""
    from deseq2_b200 import device_pipeline as DP
    N, m = K.shape
    idx = res["idx"].cpu().numpy()

    def full(v, fill=NAN):
        v = v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        a = np.full((N,) + v.shape[1:], fill)
        a[idx] = v
        return a

    dds = {k: full(res[k]) for k in ("betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue", "maxCooks", "dispersion")}
    dds["baseMean"] = full(res["baseMean"], 0.0)
    dds["allZero"] = np.ones(N, bool)
    dds["allZero"][idx] = False
    dds["sizeFactors"] = res["sizeFactors"]
    ynz = y[res["idx"]].contiguous()
    sfd = res.get("normalizationFactors")
    ck = DP.cooks(ynz, res["mu"], res["H"], x, res["sizeFactors"], normalizationFactors=sfd)["cooks"]
    cooks = full(ck[:, :m])
    if nf is not None:
        dds["normalizationFactors"] = nf
    if res.get("weights") is not None:
        dds["weights"] = res["weights"][:, :m].cpu().numpy()
        wf = res["weightsFail"].cpu().numpy()
        dds["weightsFail"] = wf
        dds["baseMean"][wf] = pipeline.getBaseMeansAndVariances(K, res["sizeFactors"], weights)["baseMean"][wf]
    if res.get("modelMatrix") is not None:
        dds["betaPriorVar"], dds["modelMatrix"] = res["betaPriorVar"], res["modelMatrix"]
    if "replace" in res:
        dds["replace"] = full(res["replace"].to(torch.float64), 0.0).astype(bool)
        newc, _, _ = pipeline.replaceOutliers(K[idx], cooks[idx], res["sizeFactors"], x, minReplicates=7)
        dds["replaceCounts"] = K.copy()
        dds["replaceCounts"][idx] = newc
    return dds, cooks


def _compare(dv, host, rel=1e-12):
    for k in ("baseMean", "log2FoldChange", "lfcSE", "stat", "pvalue", "padj"):
        a, b = dv[k].cpu().numpy(), host[k]
        assert np.array_equal(np.isnan(a), np.isnan(b)), k
        f = ~np.isnan(b)
        assert np.all(np.abs(a[f] - b[f]) <= rel * np.maximum(np.abs(b[f]), 1e-300) + (b[f] == 0) * 1e-300), k
    dm, hm = dv["metadata"], host["metadata"]
    if "j" in hm:
        assert dm["j"] == hm["j"] and dm["filterTheta"] == hm["filterTheta"]
        assert np.array_equal(dm["filterNumRej"]["numRej"], hm["filterNumRej"]["numRej"])
        assert np.array_equal(dm["filterNumRej"]["theta"], hm["filterNumRej"]["theta"])
        assert dm["filterThreshold"] == hm["filterThreshold"]


def _case(kind, dev, seed=11):
    """(K, x, factors, DESeq_device kwargs) of a named case."""
    if kind == "replace":
        factors = [np.repeat([0, 1, 2], 7)]                     # 7 replicates per cell: outliers are replaced
        x = pipeline.factorDesign(factors)[0]
        d = synth.make_example_counts(300, 21, x=x, seed=seed)
        K = d["counts"].copy()
        K[0] = np.repeat([100, 200, 400], 7)
        K[0, 9] = 20000                                          # an outlier, replaced by the cell's trimmed mean
        K[1] = 0
        K[1, 16] = 500                                           # its only count is an outlier: all zero once replaced
        K[3:6] = 0
        return K, x, factors, dict(sizeFactors=d["sizeFactors"], minReplicatesForReplace=7)
    if kind == "two_group":
        factors = [np.repeat([0, 1], 4)]
        x = pipeline.factorDesign(factors)[0]
        d = synth.make_example_counts(300, 8, x=x, seed=seed)
        K = d["counts"].copy()
        K[0] = [10, 12, 11, 400, 1000, 1100, 1050, 990]          # outlier below 4 larger counts: kept
        K[1] = [10, 12, 11, 9, 10, 11, 12, 900]                  # outlier above every other count: filtered
        K[2:5] = 0
        return K, x, factors, dict(sizeFactors=d["sizeFactors"])
    factors = [np.tile([0, 1], 6), np.repeat([0, 1, 2], 4)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(300, 12, x=x, seed=seed)
    K = d["counts"].copy()
    K[0] = np.repeat([100, 200, 800], 4)
    K[3:6] = 0
    K[7, 4:12] = 0                                              # condition 2 and 3 all zero: contrastAllZero
    return K, x, factors, dict(sizeFactors=np.ones(12) if kind == "unit_sf" else d["sizeFactors"])


def _run(dev, engine, kind, deseq_kw=None, lrt=False, **kw):
    from deseq2_b200 import device_pipeline as DP
    K, x, factors, base = _case(kind, dev)
    base.update(deseq_kw or {})
    y = gm(K, dev)
    nf, w = base.get("normalizationFactors"), base.get("weights")
    if nf is not None:
        base["normalizationFactors"] = gm(nf, dev)
    if w is not None:
        base["weights"] = gm(w, dev)
        kw = dict(kw, weights=base["weights"])
    if base.get("betaPrior"):
        base["factors"] = factors
    res = DP.DESeq_device(y, x, **base)
    dds, cooks = _host_inputs(res, y, K, x, dev, nf=nf, weights=w)
    lr, lrh = None, None
    if lrt:
        ynz = y[res["idx"]].contiguous()
        lr = DP.nbinomLRT_device(ynz, x, x[:, :2], res["sizeFactors"], res["dispersion"])
        lrh = {k: np.full(K.shape[0], NAN) for k in ("LRTStatistic", "LRTPvalue")}
        for k in lrh:
            lrh[k][res["idx"].cpu().numpy()] = lr[k].cpu().numpy()
    dv = DP.results_device(res, y, x, factors=factors, lrt=lr, **kw)
    host = pipeline.results(dds, K, x, factors=factors, lrt=lrh, cooks=cooks, engine=engine,
                            **{k: v for k, v in kw.items() if k != "weights"})
    _compare(dv, host)
    return dv, host, res


CASES = [
    ("default", {}, {}),
    ("no_filtering", {}, dict(independentFiltering=False)),
    ("BY", {}, dict(pAdjustMethod="BY")),
    ("holm", {}, dict(pAdjustMethod="holm")),
    ("hochberg", {}, dict(pAdjustMethod="hochberg")),
    ("bonferroni", {}, dict(pAdjustMethod="bonferroni")),
    ("none", {}, dict(pAdjustMethod="none", alpha=0.05)),
    ("fdr_no_filter", {}, dict(pAdjustMethod="fdr", independentFiltering=False)),
    ("greaterAbs", {}, dict(lfcThreshold=0.5)),
    ("greaterAbs2014", {}, dict(lfcThreshold=0.5, altHypothesis="greaterAbs2014")),
    ("lessAbs", {}, dict(lfcThreshold=2.0, altHypothesis="lessAbs")),
    ("greater", {}, dict(lfcThreshold=0.5, altHypothesis="greater")),
    ("less", {}, dict(lfcThreshold=0.5, altHypothesis="less")),
    ("cooks_off", {}, dict(cooksCutoff=False)),
    ("cooks_num", {}, dict(cooksCutoff=1.0)),
    ("filter_theta", {}, dict(filter=np.arange(300.0) % 37, theta=np.linspace(0.1, 0.9, 9))),
    ("contrast_level", {}, dict(contrast=(1, 1, 2))),
    ("contrast_swap", {}, dict(contrast=(1, 0, 2))),
    ("contrast_list", {}, dict(contrast=[["f12"], ["f11"]], listValues=(0.5, -0.5))),
    ("contrast_numeric", {}, dict(contrast=np.array([0.0, 1.0, -1.0, 0.0]))),
    ("nf", dict(normalizationFactors="nf"), dict(contrast=(1, 1, 2))),
    ("weights", dict(weights="w"), dict(contrast=(1, 1, 2))),
    ("betaPrior", dict(betaPrior=True), {}),
    ("betaPrior_contrast", dict(betaPrior=True), dict(contrast=(1, 0, 1))),
]


def _deseq_kw(kw, shape):
    rng = np.random.default_rng(5)
    out = dict(kw)
    if out.get("normalizationFactors") == "nf":
        out["normalizationFactors"] = np.exp(rng.normal(0, 0.2, shape))
        out["sizeFactors"] = None
    if out.get("weights") == "w":
        out["weights"] = rng.uniform(0.5, 1.0, shape)
        out["weights"][8, 8:12] = 0.0                             # condition level 2 unweighted: a weightsFail row
    return out


@pytest.mark.parametrize("case", ["default", "no_filtering", "holm", "lessAbs", "contrast_level", "contrast_swap"])
def test_results_device_matches_host_emulated(emu_dev, case):
    _, dkw, kw = next(c for c in CASES if c[0] == case)
    _run("cpu", emu_dev, "factors", _deseq_kw(dkw, (300, 12)), **kw)


def _check_replacement(dev, engine):
    """Outlier replacement with 7 replicates per cell, on the coefficient path and under a contrast (getContrast on
    the replaced counts): a replaced row whose counts are now all zero gets LFC, SE, stat 0 and p 1."""
    for kw in ({}, dict(contrast=(0, 1, 2)), dict(contrast=np.array([0.0, 1.0, -0.5]))):
        dv, host, res = _run(dev, engine, "replace", **kw)
        assert res["n_replaced"] > 0 and bool(res["replace"][0]) and bool(res["replace"][1])
        assert res["baseMean"][1].item() == 0.0
        assert [dv[k][1].item() for k in ("log2FoldChange", "lfcSE", "stat", "pvalue")] == [0.0, 0.0, 0.0, 1.0]
        assert np.isfinite(dv["pvalue"][0].item()) and np.isnan(dv["pvalue"][3].item())


def test_replacement_emulated(emu_dev):
    _check_replacement("cpu", emu_dev)


def test_weights_fail_rows_emulated(emu_dev):
    """A weightsFail row keeps its weighted baseMean (mean of w K / s) and counts in the filter; NaN elsewhere."""
    from deseq2_b200 import device_pipeline as DP
    dv, host, res = _run("cpu", emu_dev, "factors", _deseq_kw(dict(weights="w"), (300, 12)))
    assert bool(res["weightsFail"][8])
    K, _, _, kw = _case("factors", "cpu")
    w = _deseq_kw(dict(weights="w"), (300, 12))["weights"]
    want = pipeline.getBaseMeansAndVariances(K, kw["sizeFactors"], w)["baseMean"][8]
    assert abs(dv["baseMean"][8].item() - want) <= 1e-12 * want and np.isnan(dv["pvalue"][8].item())
    with pytest.raises(ValueError, match="weights="):
        DP.results_device(res, gm(K, "cpu"), _case("factors", "cpu")[1])


def test_two_group_heuristic_emulated(emu_dev):
    """Both planted outliers are flagged (cutoff 2); the one with >= 3 larger counts is kept by the heuristic, the other
    loses its p-value; without the factors there is no heuristic."""
    from deseq2_b200 import device_pipeline as DP
    dv, host, res = _run("cpu", emu_dev, "two_group", cooksCutoff=2.0)
    mc = res["maxCooks"].numpy()
    assert mc[0] > 2.0 and mc[1] > 2.0
    p = dv["pvalue"].numpy()
    assert np.isfinite(p[0]) and np.isnan(p[1])
    K, x, _, _ = _case("two_group", "cpu")
    assert np.isnan(DP.results_device(res, gm(K, "cpu"), x, cooksCutoff=2.0)["pvalue"].numpy()[0])


def test_reference_expectations_emulated(emu_dev):
    """tests/testthat/test_results.R: gene 1 with counts 100 / 200 / 800 over condition levels 1-3 (unit size factors)
    gives the contrasts -3 / -1 / -2 and the list contrast 2; contrastAllZero sets LFC, stat 0 and p 1."""
    from deseq2_b200 import device_pipeline as DP
    K, x, factors, kw = _case("unit_sf", "cpu")
    y = gm(K, "cpu")
    res = DP.DESeq_device(y, x, **kw)
    R = lambda **a: DP.results_device(res, y, x, factors=factors, **a)
    for c, want in (((1, 0, 2), -3), ((1, 0, 1), -1), ((1, 1, 2), -2)):
        assert abs(R(contrast=c)["log2FoldChange"][0].item() - want) < 1e-6
    assert abs(R(contrast=[["f12"], ["f11"]])["log2FoldChange"][0].item() - 2) < 1e-6
    r = R(contrast=(1, 1, 2))
    assert r["log2FoldChange"][7].item() == 0 and r["stat"][7].item() == 0 and r["pvalue"][7].item() == 1
    assert np.isnan(r["pvalue"][3].item()) and r["baseMean"][3].item() == 0
    with pytest.raises(ValueError):
        R(lfcThreshold=1, altHypothesis="lessAbs", lrt={"LRTStatistic": None})


def test_results_device_errors_and_abi(emu_dev):
    from deseq2_b200 import _lib, device_pipeline as DP
    K, x, factors, kw = _case("factors", "cpu")
    y = gm(K, "cpu")
    res = DP.DESeq_device(y, x, **kw)
    for bad in (dict(alpha=1.0), dict(lfcThreshold=-1), dict(altHypothesis="lessAbs"), dict(pAdjustMethod="hommel"),
                dict(theta=[0.5]), dict(filter=np.ones(5)), dict(filter=lambda r: r), dict(contrast=np.zeros(4))):
        with pytest.raises(ValueError):
            DP.results_device(res, y, x, factors=factors, **bad)
    L = _lib.lib()
    P = lambda t: C.c_void_p(t.data_ptr())
    v = torch.zeros(4, dtype=torch.float64)
    i32 = torch.zeros(4, dtype=torch.int32)
    i64 = torch.zeros(4, dtype=torch.int64)
    g = dict(y=P(y), n=4, m=12, ld=y.shape[1], col=P(v), mask=None, alt=0, T=0.0, rep=None, bm=None, out=P(v))

    def gene(**kw):
        a = dict(g, **kw)
        return L.b200nb_results_gene_dev(a["y"], 0, a["n"], a["m"], a["ld"], a["col"], P(v), P(v), P(v), 0, a["mask"],
                                         0, a["alt"], a["T"], None, 0.0, None, a["rep"], a["bm"], a["out"], P(v), P(v),
                                         P(v), None)
    assert gene() == 0 and gene(n=0) == 0
    for bad in (dict(n=-1), dict(m=0), dict(ld=11), dict(alt=6), dict(alt=-1), dict(T=-1.0), dict(T=float("inf")),
                dict(col=None), dict(out=None), dict(y=None, mask=P(i32)), dict(rep=P(i32))):
        assert gene(**bad) != 0, bad
        assert L.b200nb_last_error()
    h = lambda k=1, m=12, ld=y.shape[1], ldc=12, rows=P(i64), keep=P(i32): L.b200nb_results_heuristic_dev(
        P(y), 0, rows, k, m, ld, P(torch.zeros(12, dtype=torch.float64)), ldc, keep, None)
    assert h() == 0 and h(k=0) == 0
    for bad in (dict(k=-1), dict(m=0), dict(ld=11), dict(ldc=11), dict(rows=None), dict(keep=None)):
        assert h(**bad) != 0, bad
    cf = lambda n=4, t=2, f=P(v), out=P(v): L.b200nb_filter_cutoffs_dev(f, n, P(v), t, out, None)
    assert cf() == 0
    for bad in (dict(n=0), dict(t=0), dict(t=65536), dict(f=None), dict(out=None)):
        assert cf(**bad) != 0, bad
    nr = lambda n=4, t=2, meth=0, a=0.1, c=P(v), o=P(i32): L.b200nb_filter_numrej_dev(P(v), P(v), n, c, t, meth, a, o,
                                                                                     None)
    assert nr() == 0
    for bad in (dict(n=0), dict(t=0), dict(t=70000), dict(meth=6), dict(meth=-1), dict(a=0.0), dict(a=1.0),
                dict(a=float("nan")), dict(c=None), dict(o=None)):
        assert nr(**bad) != 0, bad
    pa = lambda n=4, j=0, meth=0, o=P(i64), out=P(v): L.b200nb_padj_dev(P(v), P(v), o, n, None, j, meth, out, None)
    assert pa() == 0
    for bad in (dict(n=0), dict(j=-1), dict(meth=7), dict(o=None), dict(out=None)):
        assert pa(**bad) != 0, bad


def test_stale_workspace_is_refused(emu_dev):
    """res["mu"] / res["H"] are DESeq_device's workspace views: after a later call with another shape the heuristic
    refuses the stale result instead of reading replaced memory."""
    from deseq2_b200 import device_pipeline as DP
    K, x, factors, kw = _case("two_group", "cpu")
    y = gm(K, "cpu")
    res = DP.DESeq_device(y, x, **kw)
    DP.results_device(res, y, x, factors=factors)
    DP.DESeq_device(gm(K[:200], "cpu"), x, **kw)
    with pytest.raises(ValueError, match="workspace"):
        DP.results_device(res, y, x, factors=factors)
    DP.results_device(res, y, x)                              # no heuristic: the views are not read


# ---------------------------------------------------------------- GPU (or the emulator with B200NB_LIB)

@pytest.mark.gpu
@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_results_device_matches_host_gpu(engine, case):
    _, dkw, kw = next(c for c in CASES if c[0] == case)
    _run(DEV, engine, "factors", _deseq_kw(dkw, (300, 12)), lrt=False, **kw)


@pytest.mark.gpu
def test_results_device_lrt_and_heuristic_gpu(engine):
    dv, host, _ = _run(DEV, engine, "factors", lrt=True)
    _run(DEV, engine, "factors", lrt=True, contrast=(0, 0, 1))        # the LRT keeps its stat under a swap
    _run(DEV, engine, "two_group")
    _run(DEV, engine, "two_group", cooksCutoff=2.0)
    _run(DEV, engine, "two_group", cooksCutoff=False)


@pytest.mark.gpu
def test_replacement_gpu(engine):
    _check_replacement(DEV, engine)


def _small(N, dev, engine, **kw):
    from deseq2_b200 import device_pipeline as DP
    rng = np.random.default_rng(N)
    pv = torch.as_tensor(rng.uniform(0, 1, N) ** 4, device=dev)
    bm = torch.as_tensor(np.where(rng.uniform(0, 1, N) < 0.3, 0.0, rng.exponential(50, N)), device=dev)
    if N > 2:
        pv[::5] = float("nan")
    padj, meta = DP.p_value_adjustment(pv, bm, **kw)
    hp, hm = pipeline.pvalueAdjustment(pv.cpu().numpy(), bm.cpu().numpy(), **kw)
    a = padj.cpu().numpy()
    assert np.array_equal(np.isnan(a), np.isnan(hp))
    assert np.allclose(a[~np.isnan(hp)], hp[~np.isnan(hp)], rtol=1e-12, atol=0)
    if "j" in hm:
        assert meta["j"] == hm["j"] and np.array_equal(meta["filterNumRej"]["numRej"], hm["filterNumRej"]["numRej"])
    return padj


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 2, 37, 20000])
@pytest.mark.parametrize("method", ["BH", "BY", "holm", "hochberg", "bonferroni", "none"])
def test_adjustment_sizes_gpu(engine, N, method):
    a = _small(N, DEV, engine, pAdjustMethod=method)
    b = _small(N, DEV, engine, pAdjustMethod=method)
    assert torch.equal(torch.nan_to_num(a, nan=-1.0), torch.nan_to_num(b, nan=-1.0))   # same bits
    _small(N, DEV, engine, pAdjustMethod=method, independentFiltering=False)


@pytest.mark.gpu
def test_adjustment_edge_cases_gpu(engine):
    from deseq2_b200 import device_pipeline as DP
    N = 500
    nanp = torch.full((N,), float("nan"), dtype=torch.float64, device=DEV)
    bm = torch.as_tensor(np.arange(N, dtype=np.float64), device=DEV)
    padj, meta = DP.p_value_adjustment(nanp, bm)                       # all p NA
    assert torch.isnan(padj).all() and meta["j"] == 0
    zero = torch.as_tensor(np.r_[np.zeros(480), np.arange(1.0, 21.0)], device=DEV)   # lo >= .95: theta up to 1
    pv = torch.as_tensor(np.random.default_rng(2).uniform(0, 1, N) ** 8, device=DEV)
    padj, meta = DP.p_value_adjustment(pv, zero)
    hp, hm = pipeline.pvalueAdjustment(pv.cpu().numpy(), zero.cpu().numpy())
    assert meta["filterNumRej"]["theta"][-1] == 1.0 and meta["j"] == hm["j"]
    assert np.allclose(padj.cpu().numpy(), hp, rtol=1e-12, equal_nan=True)
    few = torch.as_tensor(np.r_[np.full(5, 1e-6), np.full(N - 5, 0.9)], device=DEV)   # max(numRej) <= 10: R's j = 1
    padj, meta = DP.p_value_adjustment(few, bm)
    assert meta["j"] == 0 and max(meta["filterNumRej"]["numRej"]) <= 10


@pytest.mark.gpu
def test_results_device_c2_gpu(engine):
    """A C2-sized run (50 000 genes, 100 samples): device == host mirror, and two calls give the same bits."""
    from deseq2_b200 import device_pipeline as DP
    factors = [np.repeat([0, 1], 50)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(50000, 100, x=x, seed=3)
    K = d["counts"]
    y = gm(K, DEV)
    res = DP.DESeq_device(y, x, sizeFactors=d["sizeFactors"])
    dds, cooks = _host_inputs(res, y, K, x, DEV)
    dv = DP.results_device(res, y, x, factors=factors)
    _compare(dv, pipeline.results(dds, K, x, factors=factors, cooks=cooks, engine=engine))
    dv2 = DP.results_device(res, y, x, factors=factors)
    for k in ("log2FoldChange", "stat", "pvalue", "padj"):
        assert torch.equal(torch.nan_to_num(dv[k], nan=-7.0), torch.nan_to_num(dv2[k], nan=-7.0))


# ---------------------------------------------------------------- sharded

_SHARDED_CALLS = (("default", {}), ("holm", dict(pAdjustMethod="holm", cooksCutoff=2.0)),
                  ("no_filter", dict(independentFiltering=False)))


def _sharded_case(n):
    factors = [np.repeat([0, 1], 6)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(n, 12, x=x, seed=93)
    K = d["counts"].copy()
    K[[5, 250]] = 0
    K[7] = [10, 12, 11, 9, 10, 11, 12, 13, 10, 12, 11, 900]
    return K, x, factors, d["sizeFactors"]


def _sharded_rank(rank, world, dev, n):
    from deseq2_b200 import sharded
    K, x, factors, sf = _sharded_case(n)
    lo, hi = sharded.shard_bounds(n, world, rank)
    y = gm(K[lo:hi], dev)
    res = sharded.sharded_DESeq_device(y, x, sf)
    out = {}
    for name, kw in _SHARDED_CALLS:
        r = sharded.sharded_results_device(res, y, x, factors=factors, **kw)
        out[name] = {k: r[k] for k in ("baseMean", "log2FoldChange", "stat", "pvalue", "padj")}
        out[name]["j"] = r["metadata"].get("j")
        out[name]["collectives"] = r["collectives"]
    return out


def _check_sharded(backend, n, world=2):
    """results() over the ranks (one PackedGather of [filter, pvalue]) equals the unsharded results_device bit for
    bit."""
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_sharded_rank, n, world=world, backend=backend)
    K, x, factors, sf = _sharded_case(n)
    y = gm(K, DEVICE[backend])
    res = DP.DESeq_device(y, x, sf)
    for name, kw in _SHARDED_CALLS:
        whole = DP.results_device(res, y, x, factors=factors, **kw)
        for g in got:
            assert g[name]["j"] == whole["metadata"].get("j")
            assert g[name]["collectives"] == 2                    # the size agreement and the one gather
        for k in ("baseMean", "log2FoldChange", "stat", "pvalue", "padj"):
            cat = np.concatenate([g[name][k] for g in got])
            assert np.array_equal(cat, whole[k].cpu().numpy(), equal_nan=True), (name, k)


def test_sharded_results_equal_whole(emu_dev):
    _check_sharded("gloo", 401)


@pytest.mark.gpu
def test_sharded_results_over_nccl_equals_whole(engine):
    _check_sharded("nccl", 20000, nccl_world())
