"""DESeq(test = "LRT") on the device: DESeq_device(test="LRT", reduced=...) against the two-call sequence DESeq_device +
nbinomLRT_device (bit for bit), the intercept-only closed form against a numpy / scipy restatement of
R/fitNbinomGLMs.R:99-137, the device against the host mirror pipeline.DESeq(test="LRT") on the oracle engine, the LRT
refit of replaced genes, results_device on an LRT result (the applicable expectations of the reference's
test_results.R and test_LRT.R) and the gene-sharded run.  The CPU tests run the engine's CUDA source on the SIMT
emulator (`emu_dev`); the `-m gpu` tests run on a GPU, or on the emulator when B200NB_LIB points at it."""
import warnings

import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm, rel_err  # noqa: F401
from deseq2_b200 import pipeline, synth
from ranks import DEVICE, nccl_world, run_ranks

LRT_KEYS = ("LRTStatistic", "LRTPvalue", "df", "fullBetaConv", "reducedBetaConv", "reducedModelMatrix", "test")


def _same(a, b):
    """Bit equality of two results' values (tensors with NaN, numpy arrays, scalars, dicts)."""
    if isinstance(a, torch.Tensor):
        return (a.shape == b.shape and a.dtype == b.dtype
                and torch.equal(torch.nan_to_num(a, nan=-7.0), torch.nan_to_num(b, nan=-7.0)))
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b, equal_nan=True)
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    return a == b or (a != a and b != b)


def _snapshot(res):
    """A DESeq_device result with its tensors cloned: mu / H are workspace views that the next call overwrites."""
    return {k: v.clone() if isinstance(v, torch.Tensor) else v for k, v in res.items()}


def _tx_nf(counts, sf, seed):
    rng = np.random.default_rng(seed)
    nf = sf[None, :] * np.exp(rng.normal(0, 0.25, counts.shape))
    return nf / np.exp(np.log(nf).mean(axis=1, keepdims=True))


def _weights(n, m, x, seed):
    """Weights in (0.3, 1] with row 2 failing: zero weight on every sample of the last column's level."""
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.3, 1.0, (n, m))
    w[2, x[:, -1] == 1] = 0.0
    return w


def _case(kind, n=160, seed=11, m=12):
    """(counts, full, reduced, DESeq kwargs as numpy) of a named design."""
    if kind == "batch":                                       # C5-like: ~batch + condition vs ~batch
        x = synth.design_batch_condition(m, 3)
        xr = x[:, :3]
    elif kind == "intercept":                                 # ~condition vs ~1
        x = synth.design_condition(12)
        xr = np.ones((12, 1))
    else:                                                     # 7 replicates per level: outliers are replaced
        x = pipeline.factorDesign([np.repeat([0, 1, 2], 7)])[0]
        xr = np.ones((21, 1))
    d = synth.make_example_counts(n, x.shape[0], x=x, seed=seed, betaSD=0.7)
    K = d["counts"].copy()
    K[5 % n] = 0
    return K, x, xr, {"sizeFactors": d["sizeFactors"]}


def _device_kw(kw, K, x, dev):
    """DESeq_device's arguments from the numpy ones (weights / nf become gene-major tensors)."""
    out = dict(kw)
    for k in ("weights", "normalizationFactors"):
        if out.get(k) is not None:
            out[k] = gm(out[k], dev)
    return out


def _variant(variant, K, x, kw):
    kw = dict(kw)
    if variant == "nf":
        kw["normalizationFactors"] = _tx_nf(K, kw.pop("sizeFactors"), 3)
    elif variant == "weights":
        kw["weights"] = _weights(*K.shape, x, 4)
    return kw


# ---------------------------------------------------------------- composition identity

def _check_composition(dev, K, x, xr, kw):
    """DESeq_device(test="LRT") == DESeq_device followed by nbinomLRT_device on its dispersions, bit for bit; every
    key the Wald run has is the same in the LRT run."""
    from deseq2_b200 import device_pipeline as DP
    y = gm(K, dev)
    dkw = _device_kw(kw, K, x, dev)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        lrt = _snapshot(DP.DESeq_device(y, x, test="LRT", reduced=xr, **dkw))
        wald = _snapshot(DP.DESeq_device(y, x, **dkw))
    assert lrt["test"] == "LRT" and wald["test"] == "Wald"
    assert not any(k in wald for k in LRT_KEYS if k != "test")
    for k in wald:
        if k not in ("stage_ms", "test"):
            assert _same(lrt[k], wald[k]), k
    ynz = y[lrt["idx"]].contiguous()
    nf = lrt.get("normalizationFactors")
    seq = DP.nbinomLRT_device(ynz, x, xr, None if nf is not None else lrt["sizeFactors"], lrt["dispersion"],
                              weights=lrt.get("weights"), normalizationFactors=nf)
    for k in ("LRTStatistic", "LRTPvalue", "betaMatrix", "betaSE", "deviance", "reducedBetaConv"):
        assert _same(lrt[k], seq[k]), k
    assert _same(lrt["fullBetaConv"], seq["fullBetaConv"]) and lrt["df"] == seq["df"] == x.shape[1] - xr.shape[1]
    assert np.array_equal(lrt["reducedModelMatrix"], xr)
    assert torch.isfinite(lrt["LRTStatistic"]).all()
    return lrt, wald, seq


@pytest.mark.parametrize("variant", ["sf", "nf", "weights"])
def test_composition_identity_emulated(emu_dev, variant):
    K, x, xr, kw = _case("batch")
    lrt, _, _ = _check_composition("cpu", K, x, xr, _variant(variant, K, x, kw))
    if variant == "weights":
        assert bool(lrt["weightsFail"][2]) and 2 not in lrt["idx"].tolist()


def test_defaults_unchanged_emulated(emu_dev):
    """test="Wald" spelled out is the default call, and two calls give the same bits."""
    from deseq2_b200 import device_pipeline as DP
    K, x, _, kw = _case("batch")
    y = gm(K, "cpu")
    a = _snapshot(DP.DESeq_device(y, x, **kw))
    b = _snapshot(DP.DESeq_device(y, x, test="Wald", **kw))
    assert all(_same(a[k], b[k]) for k in a if k != "stage_ms")


# ---------------------------------------------------------------- the intercept-only closed form

def _closed_form_host(K, nf, disp, w=None):
    """R/fitNbinomGLMs.R:99-137 restated with numpy / scipy: beta = log(rowMeans(K / nf)) (weighted: sum(w K / nf) /
    sum(w)), logLike = rowSums(w * dnbinom(K, mu = nf e^beta, size = 1 / alpha, log = TRUE))."""
    from scipy import stats
    norm = K / nf
    beta = np.log(norm.mean(axis=1) if w is None else (w * norm).sum(axis=1) / w.sum(axis=1))
    mu = nf * np.exp(beta)[:, None]
    size = 1.0 / disp[:, None]
    lp = stats.nbinom.logpmf(K, size, size / (size + mu))
    return beta, (lp if w is None else w * lp).sum(axis=1)


@pytest.mark.parametrize("variant", ["sf", "nf", "weights"])
def test_intercept_closed_form_emulated(emu_dev, oracle, variant):
    """Reduced ~1: beta and the reduced log-likelihood equal the scipy restatement to 1e-12, the LRT statistic is built
    from them, and the host mirror pipeline.DESeq(test="LRT") agrees."""
    from deseq2_b200 import device_pipeline as DP
    K, x, xr, kw = _case("intercept")
    kw = _variant(variant, K, x, kw)
    y = gm(K, "cpu")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        res = DP.DESeq_device(y, x, test="LRT", reduced=xr, useOptim=False, **_device_kw(kw, K, x, "cpu"))
    rerun = _Rerun(oracle, K, x, useOptim=False, test="LRT", reduced=xr, **kw)
    host = rerun()
    idx = res["idx"].numpy()
    m = x.shape[0]
    ynz = y[res["idx"]].contiguous()
    nf = res.get("normalizationFactors")
    sfd = nf if nf is not None else torch.as_tensor(res["sizeFactors"])
    wn = res.get("weights")
    red = DP._intercept_only(ynz, sfd, res["dispersion"], wn, m)
    nfm = nf[:, :m].numpy() if nf is not None else np.broadcast_to(res["sizeFactors"], (len(idx), m))
    beta, ll = _closed_form_host(K[idx].astype(np.float64), nfm, res["dispersion"].numpy(),
                                 None if wn is None else wn[:, :m].numpy())
    assert np.max(rel_err(red["beta_mat"][0].numpy(), beta)) < 1e-12
    assert np.max(rel_err(red["logLike"].numpy(), ll)) < 1e-12
    llf = -0.5 * res["deviance"].numpy()
    stat = res["LRTStatistic"].numpy()
    assert np.max(np.abs(stat - 2.0 * (llf - ll)) / (1.0 + np.abs(res["deviance"].numpy()))) < 1e-12
    assert bool(res["reducedBetaConv"].all())
    _compare_host(res, host, _same_iterations(res, host, rerun))


# ---------------------------------------------------------------- device vs host mirror

def _same_iterations(dv, host, rerun):
    """The genes whose two dispersion line searches took the same number of steps on both sides.  The others must be
    rare and oracle-certified knife edges (decision margin below 4096 rounding bounds), as in
    test_norm_factors_device._compare_nf; rerun(engine) repeats the host run on another engine."""
    idx = dv["idx"].cpu().numpy()
    same = ((dv["dispGeneIter"].cpu().numpy() == host["dispGeneIter"][idx])
            & (dv["dispIter"].cpu().numpy() == host["dispIter"][idx]))
    if np.any(~same):
        from test_device_pipeline_gpu import _MarginOracle
        assert np.mean(~same) <= 0.05
        mo = _MarginOracle(rerun.engine)
        rerun(mo)
        margin = np.minimum(mo.margins[0], mo.margins[1])         # the GeneEst and MAP fits of all rows
        assert np.all(margin[~same] < 4096), (np.flatnonzero(~same)[:8], margin[~same][:8])
    return same


def _compare_host(dv, host, same, stat_tol=1e-9):
    """The LRT tolerances of test_device_pipeline_gpu.test_lrt_device_matches_host on the genes of `same` whose two
    fits converged: the statistic within stat_tol of (1 + |deviance|), p-values above 1e-12 within 1e-6 relative.
    Returns the compared mask (over dv's rows)."""
    idx = dv["idx"].cpu().numpy()
    ok = same & (host["fullBetaConv"][idx] == 1) & (host["reducedBetaConv"][idx] == 1)
    assert ok.sum() > 0.85 * len(idx)
    assert dv["fullBetaConv"].cpu().numpy()[ok].all() and dv["reducedBetaConv"].cpu().numpy()[ok].all()
    dev_ = host["deviance"][idx][ok]
    st = dv["LRTStatistic"].cpu().numpy()[ok]
    assert np.max(np.abs(st - host["LRTStatistic"][idx][ok]) / (1 + np.abs(dev_))) < stat_tol
    pv, hp = dv["LRTPvalue"].cpu().numpy()[ok], host["LRTPvalue"][idx][ok]
    big = hp > 1e-12
    assert np.max(rel_err(pv[big], hp[big])) < 1e-6
    assert dv["df"] == host["df"] and host["test"] == "LRT"
    return ok


class _Rerun:
    """pipeline.DESeq with fixed arguments on a given engine (for _same_iterations)."""

    def __init__(self, engine, *args, **kw):
        self.engine, self.args, self.kw = engine, args, kw

    def __call__(self, engine=None):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return pipeline.DESeq(*self.args, engine=engine or self.engine, **self.kw)


_HOST_CASES = {"batch": ("batch", {}), "intercept": ("intercept", {}), "weights": ("batch", {"variant": "weights"}),
               "nf": ("intercept", {"variant": "nf"}), "mean": ("batch", {"fitType": "mean"})}


def _check_host(dev, engine, name, n=160):
    from deseq2_b200 import device_pipeline as DP
    kind, extra = _HOST_CASES[name]
    extra = dict(extra)
    K, x, xr, kw = _case(kind, n=n)
    kw = _variant(extra.pop("variant", None), K, x, kw)
    kw.update(extra)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        dv = DP.DESeq_device(gm(K, dev), x, test="LRT", reduced=xr, useOptim=False, **_device_kw(kw, K, x, dev))
    rerun = _Rerun(engine, K, x, useOptim=False, test="LRT", reduced=xr, **kw)
    host = rerun()
    # with weights the GeneEst mean is an IRLS fit on both sides (no linear mu), stopped by betaTol = 1e-8: the
    # dispersions, and so the statistic, agree to that fit's accuracy rather than to rounding
    _compare_host(dv, host, _same_iterations(dv, host, rerun), 1e-8 if "weights" in kw else 1e-9)
    return dv, host


@pytest.mark.parametrize("name", sorted(_HOST_CASES))
def test_device_matches_host_emulated(emu_dev, oracle, name):
    dv, host = _check_host("cpu", oracle, name)
    if name == "weights":
        assert host["weightsFail"][2] and np.isnan(host["LRTStatistic"][2])


def _replace_case(n=120):
    """The reference's test_outlier.R:58-60 case (counts[1, 1] = 1e6, reduced ~1) with 7 replicates per level, more
    planted outliers, and a row whose only count is an outlier: all zero once replaced."""
    K, x, xr, kw = _case("replace", n=n, seed=21)
    K[2, 0] = 1000000
    K[0] = np.repeat([100, 200, 400], 7)
    K[0, 9] = 20000
    K[[10, 20, 30], [3, 9, 12]] = 40 * K[[10, 20, 30]].max(axis=1) + 500
    K[1] = 0
    K[1, 16] = 500
    return K, x, xr, dict(kw, minReplicatesForReplace=7)


def _check_replacement(dev, engine, n=120):
    """With R's default useOptim: the rows whose full IRLS fit did not converge (the all-zero-level rows) go to optim on
    both sides, which differ there (L-BFGS-B vs Newton); the comparison is over the rows the IRLS fitted."""
    from deseq2_b200 import device_pipeline as DP
    K, x, xr, kw = _replace_case(n)
    y = gm(K, dev)
    dv = _snapshot(DP.DESeq_device(y, x, test="LRT", reduced=xr, **kw))
    rerun = _Rerun(engine, K, x, test="LRT", reduced=xr, **kw)
    host = rerun()
    idx = dv["idx"].cpu().numpy()
    rep = dv["replace"].cpu().numpy()
    assert dv["n_replaced"] == host["n_replaced"] >= 5 and np.array_equal(rep, host["replace"][idx])
    assert rep[np.searchsorted(idx, [0, 1, 2, 10, 20, 30])].all()
    one = np.searchsorted(idx, 1)                              # all zero once replaced: NaN in every LRT column
    assert dv["baseMean"][one].item() == 0.0
    assert np.isnan(dv["LRTStatistic"][one].item()) and np.isnan(dv["LRTPvalue"][one].item())
    assert np.isnan(host["LRTStatistic"][1]) and np.isnan(host["LRTPvalue"][1])
    irls = (host["betaIter"][idx] < 100) & (dv["betaIter"].cpu().numpy() < 100)
    ok = _compare_host(dv, host, _same_iterations(dv, host, rerun) & irls)
    # the refit happened: the replaced rows differ from the same run without replacement
    plain = _snapshot(DP.DESeq_device(y, x, test="LRT", reduced=xr,
                                      **{k: v for k, v in kw.items() if k != "minReplicatesForReplace"}))
    moved = rep & ok
    assert moved.sum() >= 4
    assert np.all(dv["LRTStatistic"].cpu().numpy()[moved] != plain["LRTStatistic"].cpu().numpy()[moved])
    assert torch.equal(dv["LRTStatistic"][~dv["replace"]], plain["LRTStatistic"][~dv["replace"]])
    return dv


def test_replacement_refits_the_lrt_emulated(emu_dev, oracle):
    _check_replacement("cpu", oracle)


# ---------------------------------------------------------------- results()

def _results_case():
    """test_results.R:104-118: ~group + condition, reduced ~group."""
    factors = [np.tile([0, 1], 6), np.repeat([0, 1], 6)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(200, 12, x=x, seed=1, betaSD=0.7)
    K = d["counts"].copy()
    K[4] = 0
    return K, x, x[:, :2], factors, d["sizeFactors"]


def test_results_of_an_lrt_result_emulated(emu_dev):
    from deseq2_b200 import device_pipeline as DP
    K, x, xr, factors, sf = _results_case()
    y = gm(K, "cpu")
    lrt = _snapshot(DP.DESeq_device(y, x, sf, test="LRT", reduced=xr))
    wald = _snapshot(DP.DESeq_device(y, x, sf))
    R = lambda res, **a: DP.results_device(res, y, x, factors=factors, **a)
    keys = ("baseMean", "log2FoldChange", "lfcSE", "stat", "pvalue", "padj")
    # the LRT statistic is not the Wald statistic of the same column
    a, b = R(lrt, name="f11"), R(lrt, name="f11", test="Wald")
    fin = torch.isfinite(a["stat"])
    assert not torch.equal(a["stat"][fin], b["stat"][fin])
    # an LRT result gives what a Wald result with lrt= gives (no replacement), and test="Wald" the Wald results
    ynz = y[lrt["idx"]].contiguous()
    seq = DP.nbinomLRT_device(ynz, x, xr, sf, wald["dispersion"])
    for kw in ({}, dict(contrast=(1, 1, 0)), dict(pAdjustMethod="holm", independentFiltering=False)):
        got, want = R(lrt, **kw), R(wald, lrt=seq, **kw)
        assert all(_same(got[k], want[k]) for k in keys), kw
        got, want = R(lrt, test="Wald", **kw), R(wald, **kw)
        assert all(_same(got[k], want[k]) for k in keys), kw
    assert R(lrt)["metadata"]["j"] == R(wald, lrt=seq)["metadata"]["j"]
    # the contrast swap negates the LFC and keeps the LRT statistic
    s, t = R(lrt, contrast=(0, 0, 1)), R(lrt, contrast=(0, 1, 0))
    fin = torch.isfinite(s["log2FoldChange"])
    assert torch.equal(s["log2FoldChange"][fin], -t["log2FoldChange"][fin])
    assert _same(s["stat"], t["stat"]) and _same(s["stat"], R(lrt)["stat"])
    # R's stops
    with pytest.raises(ValueError, match="Wald"):
        R(lrt, lfcThreshold=1)
    with pytest.raises(ValueError, match="nbinomLRT"):
        R(wald, test="LRT")
    with pytest.raises(ValueError, match="lrt="):
        R(lrt, lrt=seq)
    with pytest.raises(ValueError, match="test"):
        R(lrt, test="t")
    R(lrt, test="Wald", lfcThreshold=1)                        # the Wald columns take a threshold


# ---------------------------------------------------------------- errors (test_LRT.R:2-12 for matrices)

def test_errors_device_and_host(emu_dev):
    from deseq2_b200 import device_pipeline as DP
    K, x, xr, kw = _case("batch", n=40)
    y = gm(K, "cpu")
    factors = [np.array([0, 1, 2] * 4), np.repeat([0, 1], 6)]
    xb = pipeline.factorDesign(factors)[0]
    rank_def = np.c_[x, x[:, 1] + x[:, 3]]                     # a linear combination of the other columns
    zero_col = np.c_[xr, np.zeros(12)]                         # a level without samples
    for bad, match in ((dict(test="LRT"), "reduced"), (dict(reduced=xr), "ignored"),
                       (dict(test="LRT", reduced=x), "columns"), (dict(test="LRT", reduced=np.c_[x, x[:, 1] ** 2 + 1]),
                                                                  "not full rank|columns"),
                       (dict(test="LRT", reduced=zero_col), "reduced model matrix is not full rank"),
                       (dict(test="LRT", reduced=xr[:10]), "one row per sample"), (dict(test="t"), "Wald"),
                       (dict(test="LRT", reduced=xb[:, :2], betaPrior=True, factors=factors, full=xb), "shrinkage"),
                       (dict(test="LRT", reduced=xr, full=rank_def), "full model matrix is not full rank")):
        bad = dict(bad)
        full = bad.pop("full", x)
        with pytest.raises(ValueError, match=match):
            DP.DESeq_device(y, full, kw["sizeFactors"], **bad)
        with pytest.raises(ValueError, match=match):
            pipeline.DESeq(K, full, sizeFactors=kw["sizeFactors"], engine=emu_dev, **bad)


# ---------------------------------------------------------------- sizes

@pytest.mark.parametrize("N", [1, 2, 37])
def test_small_sizes_emulated(emu_dev, N):
    """From one gene on, both reduced kinds; two calls give the same bits."""
    from deseq2_b200 import device_pipeline as DP
    for kind in ("batch", "intercept"):
        K, x, xr, kw = _case(kind, n=N + 6)
        K = K[K.sum(axis=1) > 0][:N]
        y = gm(K, "cpu")
        kw["fitType"] = "mean" if N < 10 else "parametric"
        a = _snapshot(DP.DESeq_device(y, x, test="LRT", reduced=xr, **kw))
        b = _snapshot(DP.DESeq_device(y, x, test="LRT", reduced=xr, **kw))
        assert a["LRTStatistic"].numel() == N
        assert all(_same(a[k], b[k]) for k in a if k != "stage_ms")
        seq = DP.nbinomLRT_device(y, x, xr, kw["sizeFactors"], a["dispersion"])
        if kind == "batch":                                    # nbinomLRT_device fits an unweighted ~1 by IRLS
            assert _same(a["LRTStatistic"], seq["LRTStatistic"])


# ---------------------------------------------------------------- sharded

def _sharded_case(n, m):
    K, x, xr, kw = _case("batch", n=n, seed=93, m=m)
    K[250] = 0
    return K, x, xr, kw["sizeFactors"]


def _sharded_rank(rank, world, dev, n, m):
    from deseq2_b200 import sharded
    K, x, xr, sf = _sharded_case(n, m)
    lo, hi = sharded.shard_bounds(n, world, rank)
    y = gm(K[lo:hi], dev)
    wald = sharded.sharded_DESeq_device(y, x, sf)
    r = sharded.sharded_DESeq_device(y, x, sf, test="LRT", reduced=xr)
    out = sharded.sharded_results_device(r, y, x)
    return {"gathered": r["gathered"], "extra_collectives": r["collectives"] - wald["collectives"],
            "results_collectives": out["collectives"], "stat": out["stat"], "padj": out["padj"]}


def _check_sharded(backend, n, m, world=2):
    """The gathered LRT results equal the unsharded run bit for bit, through the Wald run's collectives; sharded
    results() of the LRT result equals results_device of the whole."""
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_sharded_rank, n, m, world=world, backend=backend)
    K, x, xr, sf = _sharded_case(n, m)
    y = gm(K, DEVICE[backend])
    whole = DP.DESeq_device(y, x, sf, test="LRT", reduced=xr)
    wr = DP.results_device(whole, y, x)
    for g in got:
        assert g["extra_collectives"] == 0
        assert set(g["gathered"]) == {"dispersion", "betaMatrix", "betaSE", "LRTStatistic", "LRTPvalue"}
        for k, v in g["gathered"].items():
            assert np.array_equal(v, whole[k].cpu().numpy(), equal_nan=True), k
        assert g["results_collectives"] == 2
    for k in ("stat", "padj"):
        cat = np.concatenate([g[k] for g in got])
        assert np.array_equal(cat, wr[k].cpu().numpy(), equal_nan=True), k


def test_sharded_lrt_equals_whole(emu_dev):
    _check_sharded("gloo", 301, 12)


# ---------------------------------------------------------------- GPU (or the emulator with B200NB_LIB)

@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["sf", "nf", "weights"])
def test_composition_identity_gpu(engine, variant):
    K, x, xr, kw = _case("batch", n=3000)
    _check_composition(DEV, K, x, xr, _variant(variant, K, x, kw))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_HOST_CASES))
def test_device_matches_host_gpu(engine, oracle, name):
    _check_host(DEV, oracle, name, n=1500)


@pytest.mark.gpu
def test_replacement_refits_the_lrt_gpu(engine, oracle):
    _check_replacement(DEV, oracle, n=600)


@pytest.mark.gpu
@pytest.mark.parametrize("reduced", ["condition", "intercept"])
def test_c2_size_gpu(engine, reduced):
    """50 000 x 100: the one-call LRT equals the two-call sequence (~batch + condition vs ~batch) or is finite with
    the closed form (~condition vs ~1), and two calls give the same bits."""
    from deseq2_b200 import device_pipeline as DP
    n = 50000 if DEV == "cuda" else 500
    x = synth.design_batch_condition(100, 2) if reduced == "condition" else synth.design_condition(100)
    xr = x[:, :2] if reduced == "condition" else np.ones((100, 1))
    d = synth.make_example_counts(n, 100, x=x, seed=3)
    y = gm(d["counts"], DEV)
    a = _snapshot(DP.DESeq_device(y, x, d["sizeFactors"], test="LRT", reduced=xr))
    b = _snapshot(DP.DESeq_device(y, x, d["sizeFactors"], test="LRT", reduced=xr))
    assert all(_same(a[k], b[k]) for k in a if k != "stage_ms")
    assert torch.isfinite(a["LRTStatistic"]).all() and ((a["LRTPvalue"] >= 0) & (a["LRTPvalue"] <= 1)).all()
    if reduced == "condition":
        ynz = y[a["idx"]].contiguous()
        seq = DP.nbinomLRT_device(ynz, x, xr, d["sizeFactors"], a["dispersion"])
        for k in ("LRTStatistic", "LRTPvalue", "betaMatrix", "betaSE", "deviance"):
            assert _same(a[k], seq[k]), k


@pytest.mark.gpu
def test_sharded_lrt_over_nccl_equals_whole(engine):
    _check_sharded("nccl", 20000, 60, nccl_world())
