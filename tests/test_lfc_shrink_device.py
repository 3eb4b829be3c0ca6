"""lfcShrink(type = "normal") on the device (device_pipeline.lfcShrink_device): the standard-matrix prior variance
(b200nb_beta_prior_quantile_dev, one quantile per non-intercept column) against the host restatement of
estimateBetaPriorVar, the whole call against the host mirror pipeline.lfcShrink fed the same DESeq_device result,
identities that need no mirror (untouched columns, DESeq(betaPrior=TRUE) for factor-level contrasts, the penalised
score of the MAP fit), R's stops, and the gene-sharded call.  The CPU tests run the engine's CUDA source on the SIMT
emulator (`emu_dev` fixture); the `-m gpu` tests run on a GPU, or on the emulator when B200NB_LIB points at it."""
import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm, rel_err
from deseq2_b200 import pipeline, synth
from ranks import DEVICE, nccl_world, run_ranks

NAN = np.nan
COLS = ("baseMean", "log2FoldChange", "lfcSE", "stat", "pvalue", "padj")
LN2 = float(np.log(2.0))


# ---------------------------------------------------------------- the standard-matrix prior variance

def _inputs(n, p, seed, sd=1.5):
    rng = np.random.default_rng(seed)
    beta = rng.normal(0.0, sd, (n, p))
    baseMean = np.exp(rng.normal(4.0, 2.0, n))
    return beta, baseMean, 0.05 + 2.0 / baseMean


def _check_standard_prior(beta, bm, df, dev="cpu"):
    from deseq2_b200 import device_pipeline as DP
    T = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    pv = DP.estimate_beta_prior_var(T(beta), None, T(bm), T(df), expandedType=False).cpu().numpy()
    p = beta.shape[1]
    names = ["Intercept"] + [f"c{j}" for j in range(1, p)]
    ref, _ = pipeline.estimateBetaPriorVar(beta, names, np.r_[-1, np.zeros(p - 1, int)], bm, df, expandedType=False)
    assert pv.shape == (p,) and pv[0] == 1e6
    assert np.all(rel_err(pv, ref, floor=1e-300) <= 1e-12), (pv, ref)
    return pv


@pytest.mark.parametrize("n", [1, 2, 7, 999, 20000])
def test_standard_prior_matches_host_random(emu_dev, n):
    _check_standard_prior(*_inputs(n, 4, seed=n))


def test_standard_prior_wide_column_and_single_gene(emu_dev):
    beta, bm, df = _inputs(500, 3, seed=4)
    beta[:, 2] = np.where(np.arange(500) % 2 == 0, 10.0, -25.0)      # no |beta| < 10: the wide prior
    pv = _check_standard_prior(beta, bm, df)
    assert pv[2] == 1e6 and pv[1] < 1e6
    one, bm1, df1 = _inputs(1, 4, seed=5)
    pv1 = _check_standard_prior(one, bm1, df1)
    assert np.array_equal(pv1[1:], one[0, 1:] ** 2)                  # one gene: beta^2, no quantile


def test_standard_prior_heavy_ties(emu_dev):
    beta, bm, df = _inputs(5000, 4, seed=3, sd=0.3)
    _check_standard_prior(np.round(beta, 2), bm, df)
    _check_standard_prior(np.round(beta, 1), np.full(5000, 50.0), np.full(5000, 0.1))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 7, 999, 20000])
def test_standard_prior_matches_host_gpu(engine, n):
    beta, bm, df = _inputs(n, 5, seed=n + 7)
    beta[::13, 3] = 12.0
    _check_standard_prior(beta, bm, df, DEV)
    _check_standard_prior(np.round(beta, 1), bm, df, DEV)


# ---------------------------------------------------------------- device vs host mirror

def _case(kind, seed=11):
    """(K, x, factors, DESeq_device kwargs) of a named design."""
    rng = np.random.default_rng(seed)
    if kind == "replace":
        factors = [np.repeat([0, 1, 2], 7)]                          # 7 replicates per cell: outliers are replaced
        x = pipeline.factorDesign(factors)[0]
        d = synth.make_example_counts(300, 21, x=x, seed=seed)
        K = d["counts"].copy()
        K[0] = np.repeat([100, 200, 400], 7)
        K[0, 9] = 20000                                              # an outlier, replaced by the cell's trimmed mean
        K[1] = 0
        K[1, 16] = 500                                               # its only count is an outlier: all zero once replaced
        K[3:6] = 0
        return K, x, factors, dict(sizeFactors=d["sizeFactors"], minReplicatesForReplace=7)
    if kind == "condition":
        factors = [np.repeat([0, 1], 6)]
    elif kind == "factor3":
        factors = [np.repeat([0, 1, 2], 4)]
    elif kind == "covariate":
        factors = None
    else:                                                            # batch + condition
        factors = [np.tile([0, 1], 6), np.repeat([0, 1, 2], 4)]
    if factors is None:
        x = np.c_[np.ones(12), np.repeat([0.0, 1.0], 6), np.linspace(-1.0, 1.5, 12)]
    else:
        x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(300, 12, x=x, seed=seed)
    K = d["counts"].copy()
    K[3:6] = 0
    K[7, 4:12] = 0
    kw = dict(sizeFactors=d["sizeFactors"])
    return K, x, factors, kw


def _host_dds(res, y, K, x, nf=None, weights=None):
    """pipeline.DESeq's layout (all N rows) from a DESeq_device result, and the first fit's Cook's matrix."""
    from deseq2_b200 import device_pipeline as DP
    N, m = K.shape
    idx = res["idx"].cpu().numpy()

    def full(v, fill=NAN):
        v = v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        a = np.full((N,) + v.shape[1:], fill)
        a[idx] = v
        return a

    keys = ["betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue", "maxCooks", "dispersion", "dispFit"]
    if res["test"] == "LRT":
        keys += ["LRTStatistic", "LRTPvalue"]
    dds = {k: full(res[k]) for k in keys}
    dds["test"] = res["test"]
    dds["baseMean"] = full(res["baseMean"], 0.0)
    dds["allZero"] = np.ones(N, bool)
    dds["allZero"][idx] = False
    dds["sizeFactors"] = res["sizeFactors"]
    ynz = y[res["idx"]].contiguous()
    ck = DP.cooks(ynz, res["mu"], res["H"], x, res["sizeFactors"], normalizationFactors=res.get("normalizationFactors"))
    cooks = full(ck["cooks"][:, :m])
    if nf is not None:
        dds["normalizationFactors"] = nf
    if res.get("weights") is not None:
        dds["weights"] = res["weights"][:, :m].cpu().numpy()
        wf = res["weightsFail"].cpu().numpy()
        dds["weightsFail"] = wf
        dds["baseMean"][wf] = pipeline.getBaseMeansAndVariances(K, res["sizeFactors"], weights)["baseMean"][wf]
    if "replace" in res:
        dds["replace"] = full(res["replace"].to(torch.float64), 0.0).astype(bool)
        newc, _, _ = pipeline.replaceOutliers(K[idx], cooks[idx], res["sizeFactors"], x, minReplicates=7)
        dds["replaceCounts"] = K.copy()
        dds["replaceCounts"][idx] = newc
    return dds, cooks


def _compare(dv, host, tol=1e-6):
    for k in COLS:
        a, b = dv[k].cpu().numpy(), host[k]
        assert np.array_equal(np.isnan(a), np.isnan(b)), k
        f = ~np.isnan(b)
        if k in ("pvalue", "padj"):
            assert np.all(np.abs(a[f] - b[f]) <= tol), (k, np.max(np.abs(a[f] - b[f])))
        else:
            assert np.all(rel_err(a[f], b[f], floor=1e-6) <= tol), (k, np.max(rel_err(a[f], b[f], floor=1e-6)))
    assert np.all(rel_err(dv["metadata"]["priorInfo"]["betaPriorVar"], host["metadata"]["priorInfo"]["betaPriorVar"],
                          floor=1e-300) <= 1e-12)


def _run(dev, engine, kind, deseq_kw=None, **kw):
    """DESeq_device on a named design, then lfcShrink_device and pipeline.lfcShrink on the same result."""
    from deseq2_b200 import device_pipeline as DP
    K, x, factors, base = _case(kind)
    base.update(deseq_kw or {})
    rng = np.random.default_rng(5)
    nf = w = None
    if base.pop("nf", False):
        nf = np.exp(rng.normal(0, 0.2, K.shape))
        base["normalizationFactors"], base["sizeFactors"] = gm(nf, dev), None
    if base.pop("w", False):
        w = rng.uniform(0.5, 1.0, K.shape)
        w[8, 8:12] = 0.0                                             # condition level 2 unweighted: a weightsFail row
        base["weights"] = gm(w, dev)
        kw = dict(kw, weights=base["weights"])
    if base.get("test") == "LRT":
        base["reduced"] = x[:, :-1]
    y = gm(K, dev)
    res = DP.DESeq_device(y, x, **base)
    dds, cooks = _host_dds(res, y, K, x, nf=nf, weights=w)
    given = kw.pop("given", None)                                    # the selection of a results table passed in
    hkw = {k: v for k, v in kw.items() if k != "weights"}
    host_res = None
    if given is not None:
        kw["results"] = DP.results_device(res, y, x, factors=factors, **given)
        host_res = pipeline.results(dds, K, x, factors=factors, cooks=cooks, engine=engine, **given)
    dv = DP.lfcShrink_device(res, y, x, factors=factors, **kw)
    host = pipeline.lfcShrink(dds, K, x, factors=factors, res=host_res, engine=engine, cooks=cooks, **hkw)
    _compare(dv, host)
    return dv, host, res, (K, x, factors, y)


CASES = [
    ("coef_condition", "condition", {}, dict(coef=1)),
    ("coef_factor3_mid", "factor3", {}, dict(coef="f01")),
    ("coef_batch_condition", "batch", {}, dict(coef=1)),
    ("coef_covariate", "covariate", {}, dict(coef=2)),
    ("contrast_ref", "batch", {}, dict(contrast=(1, 2, 0))),
    ("contrast_noref", "batch", {}, dict(contrast=(1, 1, 2))),
    ("contrast_list", "batch", {}, dict(contrast=[["f12"], ["f11"]])),
    ("contrast_numeric", "batch", {}, dict(contrast=np.array([0.0, 0.0, 0.0, 0.5, 0.5, -1.0]),
                                                  given=dict(contrast=np.array([0.0, 0.0, -0.5, 0.5])))),
    ("threshold_coef", "batch", {}, dict(coef=3, lfcThreshold=0.5)),
    ("threshold_contrast", "batch", {}, dict(contrast=(1, 1, 2), lfcThreshold=0.5)),
    ("nf_coef", "batch", dict(nf=True), dict(coef=3)),
    ("nf_contrast", "batch", dict(nf=True), dict(contrast=(1, 1, 2))),
    ("weights_coef", "batch", dict(w=True), dict(coef=3)),
    ("lrt_coef", "batch", dict(test="LRT"), dict(coef=3)),
    ("fit_type_mean", "factor3", dict(fitType="mean"), dict(coef=2)),
    ("poscounts", "factor3", dict(sizeFactors=None, sfType="poscounts"), dict(coef=2)),
]
EMULATED_CASES = ["coef_condition", "coef_covariate", "contrast_noref", "contrast_numeric", "threshold_coef",
                  "weights_coef", "lrt_coef"]


@pytest.mark.parametrize("case", EMULATED_CASES)
def test_lfc_shrink_matches_host_emulated(emu_dev, case):
    _, kind, dkw, kw = next(c for c in CASES if c[0] == case)
    _run("cpu", emu_dev, kind, dict(dkw), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_lfc_shrink_matches_host_gpu(engine, case):
    _, kind, dkw, kw = next(c for c in CASES if c[0] == case)
    _run(DEV, engine, kind, dict(dkw), **kw)


def _check_replacement(dev, engine):
    """An outlier-refit result: the MAP fit on the original counts, a row all zero once replaced gets log2FoldChange and
    lfcSE 0 (nowZero); with lfcThreshold > 0 the first fit's un-zeroed maxCooks drives the Cook's cutoff."""
    for kw in (dict(coef=2), dict(coef=2, lfcThreshold=0.3), dict(contrast=(0, 1, 2)),
               dict(contrast=(0, 2, 0), lfcThreshold=0.3)):
        dv, host, res, _ = _run(dev, engine, "replace", **kw)
        assert res["n_replaced"] > 0 and bool(res["replace"][1]) and res["baseMean"][1].item() == 0.0
        assert dv["log2FoldChange"][1].item() == 0.0 and dv["lfcSE"][1].item() == 0.0
        assert torch.isnan(dv["shrinkFit"]["betaMatrix"][1]).all()   # not fitted
        assert np.isfinite(dv["log2FoldChange"][0].item())


def test_replacement_emulated(emu_dev):
    _check_replacement("cpu", emu_dev)


@pytest.mark.gpu
def test_replacement_gpu(engine):
    _check_replacement(DEV, engine)


# ---------------------------------------------------------------- identities without the mirror

def _check_identities(dev):
    from deseq2_b200 import device_pipeline as DP
    K, x, factors, kw = _case("batch")
    y = gm(K, dev)
    res = DP.DESeq_device(y, x, **kw)
    eq = lambda a, b: torch.equal(torch.nan_to_num(a, nan=-7.0), torch.nan_to_num(b, nan=-7.0))
    # lfcThreshold = 0: every column but log2FoldChange / lfcSE is the input table's
    for sel in (dict(coef=3), dict(contrast=(1, 1, 2))):
        tab = DP.results_device(res, y, x, factors=factors, **{"name" if "coef" in sel else "contrast": v
                                                               for v in sel.values()})
        out = DP.lfcShrink_device(res, y, x, factors=factors, results=tab, **sel)
        for k in ("baseMean", "stat", "pvalue", "padj"):
            assert out[k] is tab[k], k
        assert not eq(out["log2FoldChange"], tab["log2FoldChange"])
    # a factor-level contrast: DESeq(betaPrior=TRUE) + results() computes the same numbers, bit for bit
    bp = DP.DESeq_device(y, x, betaPrior=True, factors=factors, **kw)
    for c in ((1, 1, 2), (1, 2, 0), (0, 0, 1)):
        want = DP.results_device(bp, y, x, factors=factors, contrast=c)
        got = DP.lfcShrink_device(res, y, x, factors=factors, contrast=c)
        assert np.array_equal(got["metadata"]["priorInfo"]["betaPriorVar"], bp["betaPriorVar"])
        for k in ("log2FoldChange", "lfcSE"):
            assert eq(got[k], want[k]), (c, k)
    # the penalised score of the MAP coefficients vanishes on converged rows whose means stay above minmu
    out = DP.lfcShrink_device(res, y, x, factors=factors, coef=3)
    pv = out["metadata"]["priorInfo"]["betaPriorVar"]
    sf = res["sizeFactors"]
    idx = res["idx"].cpu().numpy()
    B = out["shrinkFit"]["betaMatrix"].cpu().numpy() * LN2                  # natural log
    conv = out["shrinkFit"]["betaConv"].cpu().numpy()
    a = res["dispersion"].cpu().numpy()
    Y = K[idx].astype(np.float64)
    mu = sf[None, :] * np.exp(B @ x.T)
    ok = conv & np.all(mu > 0.5, axis=1)
    assert ok.mean() > 0.9
    r = (Y - mu) / (1.0 + a[:, None] * mu)
    lam = 1.0 / (LN2 ** 2 * pv)
    score = r @ x - lam[None, :] * B
    scale = np.abs(Y / (1.0 + a[:, None] * mu)) @ np.abs(x) + lam[None, :] * np.abs(B) + 1.0
    # the IRLS stops on a relative deviance change of betaTol: the score is zero to about sqrt(betaTol), while the
    # penalty alone is far larger on the shrunk columns
    assert np.max(np.abs(score[ok]) / scale[ok]) < 1e-4
    assert np.median(np.abs(score[ok]) / scale[ok]) < 1e-7
    assert np.max(np.abs(lam[None, 1:] * B[ok][:, 1:]) / scale[ok][:, 1:]) > 1e-2


def test_identities_emulated(emu_dev):
    _check_identities("cpu")


@pytest.mark.gpu
def test_identities_gpu(engine):
    _check_identities(DEV)


# ---------------------------------------------------------------- R's stops

def test_errors(emu_dev):
    from deseq2_b200 import device_pipeline as DP
    K, x, factors, kw = _case("batch")
    y = gm(K, "cpu")
    res = DP.DESeq_device(y, x, **kw)
    S = lambda r=res, xx=x, **a: DP.lfcShrink_device(r, y, xx, **a)
    cases = [
        (dict(coef=1, type="apeglm"), "apeglm package, which is not part of DESeq2"),
        (dict(coef=1, type="ashr"), "ashr package, which is not part of DESeq2"),
        (dict(coef=1, type="laplace"), "type must be one of"),
        (dict(factors=factors), "requires either 'coef' or 'contrast'"),
        (dict(coef=1, contrast=(1, 1, 2), factors=factors), "not both"),
        (dict(contrast=np.array([0, 0, 0, 0.5, 0.5, -1.0]), factors=factors), "user must provide 'res'"),
        (dict(coef=1, lfcThreshold=-0.5), "lfcThreshold"),
        (dict(coef=1, xx=x[:, [1, 0, 2, 3]]), "intercept"),
        (dict(contrast=(1, 1, 2)), "design factors"),
        (dict(contrast=(1, 1, 2), factors=[factors[1], factors[0]]), "only with 'coef'"),
        (dict(contrast=(1, 1, 2), factors=factors, weights=gm(np.ones(K.shape), "cpu")), "weights"),
        (dict(coef="nope", factors=factors), "not a column"),
    ]
    for a, msg in cases:
        with pytest.raises(ValueError, match=msg):
            S(**a)
    bp = DP.DESeq_device(y, x, betaPrior=True, factors=factors, **kw)
    with pytest.raises(ValueError, match="betaPrior=FALSE"):
        S(r=bp, coef=1)
    for a, msg in cases[:9]:                                         # the host mirror stops alike
        a = dict(a)
        xx = a.pop("xx", x)
        with pytest.raises(ValueError, match=msg):
            pipeline.lfcShrink({"allZero": np.zeros(len(K), bool)}, K, xx, **a)
    # a stale workspace is refused where the first fit's mu / H are read
    Kr, xr, fr, kwr = _case("replace")
    yr = gm(Kr, "cpu")
    rr = DP.DESeq_device(yr, xr, **kwr)
    DP.DESeq_device(gm(Kr[:200], "cpu"), xr, **kwr)
    with pytest.raises(ValueError, match="workspace"):
        DP.lfcShrink_device(rr, yr, xr, coef=2, lfcThreshold=0.5)


# ---------------------------------------------------------------- sharded

_SHARDED_CALLS = (("coef", dict(coef=3)), ("contrast", dict(contrast=(1, 1, 2))),
                  ("threshold", dict(coef=2, lfcThreshold=0.4)))


def _sharded_case(n):
    factors = [np.tile([0, 1], 6), np.repeat([0, 1, 2], 4)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(n, 12, x=x, seed=93)
    K = d["counts"].copy()
    K[[5, 250]] = 0
    return K, x, factors, d["sizeFactors"]


def _sharded_rank(rank, world, dev, n):
    from deseq2_b200 import sharded
    K, x, factors, sf = _sharded_case(n)
    lo, hi = sharded.shard_bounds(n, world, rank)
    y = gm(K[lo:hi], dev)
    res = sharded.sharded_DESeq_device(y, x, sf)
    out = {}
    for name, kw in _SHARDED_CALLS:
        r = sharded.sharded_lfcShrink_device(res, y, x, factors=factors, **kw)
        out[name] = {k: r[k] for k in COLS}
        out[name]["betaPriorVar"] = r["metadata"]["priorInfo"]["betaPriorVar"]
        out[name]["collectives"] = r["collectives"]
    return out


def _check_sharded(backend, n, world=2):
    """The prior over every rank's rows (one packed gather), the default table and the thresholded table (one gather
    each): the shards' rows equal the unsharded call bit for bit."""
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_sharded_rank, n, world=world, backend=backend)
    K, x, factors, sf = _sharded_case(n)
    y = gm(K, DEVICE[backend])
    res = DP.DESeq_device(y, x, sf)
    for name, kw in _SHARDED_CALLS:
        whole = DP.lfcShrink_device(res, y, x, factors=factors, **kw)
        for g in got:
            assert np.array_equal(g[name]["betaPriorVar"], whole["metadata"]["priorInfo"]["betaPriorVar"])
            # the size agreement, the prior's gather, the default table's gather and the thresholded table's
            assert g[name]["collectives"] == 3 + (kw.get("lfcThreshold", 0) > 0)
        for k in COLS:
            cat = np.concatenate([g[name][k] for g in got])
            assert np.array_equal(cat, whole[k].cpu().numpy(), equal_nan=True), (name, k)


def test_sharded_lfc_shrink_equals_whole(emu_dev):
    _check_sharded("gloo", 401)


@pytest.mark.gpu
def test_sharded_lfc_shrink_over_nccl_equals_whole(engine):
    _check_sharded("nccl", 20000, nccl_world())
