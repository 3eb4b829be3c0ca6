"""DESeq() with observation weights on the device: the weighted prep kernel (b200nb_prep_weighted_dev,
csrc/pipeline_kernels.cu) against the host restatement of getAndCheckWeights / getBaseMeansAndVariances (pipeline.py,
with its numpy restatement of LINPACK dqrdc2), DESeq_device / nbinomLRT_device / getContrast_device with weights
against pipeline.DESeq / nbinomLRT / getContrast driving the same engine, properties of the reference's
test_weights.R, and the gene-sharded run.
The CPU tests run the engine's CUDA source on the SIMT emulator (`emu` fixture); the `-m gpu` tests run on a GPU, or on
the emulator when B200NB_LIB points at it."""
import warnings

import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm, gm64, rel_err
from ranks import DEVICE, nccl_world, run_ranks


def _continuous(m, seed=3):
    """[1, t, s]: covariates on a 1/8 grid (exact in binary), m distinct rows; s = 1 + 2 t exactly on the first half
    of the samples."""
    rng = np.random.default_rng(seed)
    t = rng.permutation(m) / 8.0
    s = rng.integers(0, 96, m) / 8.0
    s[: m // 2] = 1.0 + 2.0 * t[: m // 2]
    return np.c_[np.ones(m), t, s]


def _make(n, x, seed):
    from deseq2_b200 import synth
    return synth.make_example_counts(n, x.shape[0], x=x, seed=seed, betaSD=0.3)


def _host_prep(counts, x, sf, w, minDisp=1e-8, thr=1e-2):
    from deseq2_b200 import pipeline
    wn, fail = pipeline.getAndCheckWeights(w, x, thr)
    mv = pipeline.getBaseMeansAndVariances(counts, sf, w)
    m = x.shape[0]
    norm = counts / sf[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        rough = pipeline.roughDispEstimate(norm, x)
        moments = pipeline.momentsDispEstimate(mv["baseMean"], mv["baseVar"], sf)
    a0 = np.fmin(np.fmax(minDisp, np.fmin(rough, moments)), max(10, m))   # the kernel's fmin / fmax NaN rules
    return wn, fail, mv, a0


def _check_prep(counts, x, sf, w, dev="cpu", expect_fail=None):
    from deseq2_b200 import device_pipeline as DP
    y = gm64(counts, dev)
    pr = DP.prep(y, x, sf, want_mu=False, weights=gm64(w, dev))
    m = x.shape[0]
    assert int(pr["status"].item()) == 0
    wn, fail, mv, a0 = _host_prep(counts, x, sf, w)
    got_wn = pr["weightsNorm"].cpu().numpy()
    assert np.array_equal(got_wn[:, :m], wn)                          # the same division: bit for bit
    assert np.all(got_wn[:, m:] == 0.0)
    assert np.array_equal(pr["weightsFail"].cpu().numpy() != 0, fail)
    assert np.max(rel_err(pr["baseMean"].cpu().numpy(), mv["baseMean"])) < 1e-12
    assert np.max(rel_err(pr["baseVar"].cpu().numpy(), mv["baseVar"])) < 1e-12
    assert np.max(rel_err(pr["alpha0"].cpu().numpy(), a0)) < 1e-12
    assert np.array_equal(pr["allZero"].cpu().numpy() != 0, mv["allZero"])
    if expect_fail is not None:
        assert np.array_equal(np.flatnonzero(fail), np.asarray(expect_fail)), np.flatnonzero(fail)
    return pr


# both prep kernels: m * p >= 1024 takes the grouped kernel for factor designs, shorter rows the per-sample one
_DESIGNS = {"condition12": lambda: __import__("deseq2_b200.synth").synth.design_condition(12),
            "condition600": lambda: __import__("deseq2_b200.synth").synth.design_condition(600),
            "batch_condition36": lambda: __import__("deseq2_b200.synth").synth.design_batch_condition(36, 3),
            "batch_condition300": lambda: __import__("deseq2_b200.synth").synth.design_batch_condition(300, 3),
            "factor6_40": lambda: __import__("deseq2_b200.synth").synth.design_factor(40, 6),
            "continuous50": lambda: _continuous(50)}


@pytest.mark.parametrize("design", sorted(_DESIGNS))
def test_prep_all_ones_equals_unweighted(emu_dev, design):
    from deseq2_b200 import device_pipeline as DP, synth
    x = _DESIGNS[design]()
    d = _make(60, x, 5)
    y = gm64(d["counts"], "cpu")
    pw = DP.prep(y, x, d["sizeFactors"], want_mu=False, weights=torch.ones_like(y))
    pu = DP.prep(y, x, d["sizeFactors"], want_mu=False)
    for k in ("baseMean", "baseVar", "alpha0", "allZero", "beta0"):
        assert torch.equal(pw[k], pu[k]), k
    assert not pw["weightsFail"].any()


@pytest.mark.parametrize("design", sorted(_DESIGNS))
def test_prep_random_weights_with_zeros(emu_dev, design):
    from deseq2_b200 import synth
    x = _DESIGNS[design]()
    m = x.shape[0]
    d = _make(80, x, 7)
    counts = d["counts"].astype(np.float64)
    counts[3] = 0.0                                                    # an all-zero row
    rng = np.random.default_rng(11)
    w = rng.uniform(0.0, 3.0, counts.shape)
    w[rng.random(counts.shape) < 0.3] = 0.0
    w[:, 0] = np.maximum(w[:, 0], 0.5)                                 # every row keeps a positive weight
    _check_prep(counts, x, d["sizeFactors"], w)


def test_prep_r_zero_level_case_fails(emu_dev):
    """R's test_weights.R: w[1, 1:6] <- 0 on ~condition with m = 12 zeroes one whole level of gene 1."""
    from deseq2_b200 import synth
    x = synth.design_condition(12)
    d = _make(20, x, 2)
    w = np.ones((20, 12))
    w[0, :6] = 0.0
    w[1, :5] = 0.0                                                     # one sample of the level left: passes
    _check_prep(d["counts"], x, d["sizeFactors"], w, expect_fail=[0])


@pytest.mark.parametrize("m", [36, 300])
def test_prep_zero_weight_on_a_level(emu_dev, m):
    from deseq2_b200 import synth
    x = synth.design_batch_condition(m, 3)
    d = _make(30, x, 4)
    w = np.random.default_rng(1).uniform(0.2, 1.0, (30, m))
    w[2, x[:, 1] == 1] = 0.0                                           # batch 2 has no weight: rank(w X) < p
    w[5, x[:, 3] == 1] = 0.0                                           # condition B likewise
    ref = (x[:, 1] == 0) & (x[:, 2] == 0)
    w[7, ref] = 0.005                 # reference batch below the threshold: the intercept is b2 + b3 there, test 2 fails
    w[9, x[:, 2] == 1] = 0.005        # batch 3 below it: its column is all zero on the kept samples and is dropped
    w[11, ref] = 0.02                 # above the threshold after the normalisation: passes
    _check_prep(d["counts"], x, d["sizeFactors"], w, expect_fail=[2, 5, 7])


def test_prep_weights_below_threshold_on_a_level(emu_dev):
    from deseq2_b200 import synth
    x = synth.design_factor(40, 6)
    d = _make(24, x, 8)
    w = np.ones((24, 40))
    lvl = (np.arange(40) * 6) // 40
    w[4, lvl == 0] = 1e-3                                              # reference level below: test 2 fails
    w[6, lvl == 3] = 0.0                                               # a zero column of w X: test 1 fails
    w[8, lvl == 5] = 0.0099                                            # level column dropped in test 2: passes
    w[10, lvl == 0] = 0.0101                                           # just above the threshold: passes
    _check_prep(d["counts"], x, d["sizeFactors"], w, expect_fail=[4, 6])


def test_prep_continuous_covariates_and_collinear_subset(emu_dev):
    from deseq2_b200 import synth
    m = 50
    x = _continuous(m)
    assert len({tuple(r) for r in x}) > 32
    d = _make(40, x, 9)
    rng = np.random.default_rng(3)
    w = rng.uniform(0.1, 1.0, (40, m))
    w[1, m // 2:] = 0.0                                                # only s = 1 + 2t left: exactly collinear
    w[2, m // 2:] = 1e-3                                               # the same for test 2 only
    w[3, :] = 1e-4
    w[3, 0] = 1.0                                                      # one sample above the threshold
    w[4, ::2] = 0.0                                                    # half the samples: still full rank
    _check_prep(d["counts"], x, d["sizeFactors"], w, expect_fail=[1, 2, 3])


def test_dqrdc2_restatement():
    """The host rank routine against numpy's SVD rank on clear cases, and dqrdc2's pivoting rule on a small one."""
    from deseq2_b200 import pipeline
    rng = np.random.default_rng(0)
    for shape in ((12, 2), (40, 6), (5, 7), (1, 3)):
        z = rng.normal(size=shape)
        assert pipeline.dqrdc2_rank(z) == np.linalg.matrix_rank(z)
    z = rng.normal(size=(10, 3))
    z = np.c_[z, z[:, 0] + z[:, 1], np.zeros(10)]
    assert pipeline.dqrdc2_rank(z) == 3
    z[:, 3] += 1e-6 * rng.normal(size=10)                               # norm ratio ~1e-6 > tol: counted
    assert pipeline.dqrdc2_rank(z) == 4
    assert pipeline.dqrdc2_rank(np.zeros((4, 0))) == 0


# ---------------------------------------------------------------- argument errors

def test_weight_errors_device_and_host(emu_dev):
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    x = synth.design_condition(12)
    d = _make(30, x, 2)
    y = D.to_gene_major(d["counts"], torch.device("cpu"))
    bad = {}
    for name, (i, j, v) in {"negative": (3, 4, -0.1), "nan": (5, 0, np.nan), "inf": (6, 2, np.inf)}.items():
        w = np.ones((30, 12))
        w[i, j] = v
        bad[name] = w
    w = np.ones((30, 12))
    w[7] = 0.0
    bad["all_zero_row"] = w
    for name, w in bad.items():
        with pytest.raises(ValueError):
            DP.DESeq_device(y, x, d["sizeFactors"], weights=gm64(w, "cpu"))
        with pytest.raises(ValueError):
            pipeline.DESeq(d["counts"], x, sizeFactors=d["sizeFactors"], engine=emu_dev, weights=w)
    ok = np.ones((30, 12))
    for shape in ((29, 12), (30, 16)):
        with pytest.raises(ValueError):
            DP.DESeq_device(y, x, d["sizeFactors"], weights=torch.ones(shape, dtype=torch.float64))
    with pytest.raises(ValueError):
        DP.DESeq_device(y, x, d["sizeFactors"], weights=gm64(ok, "cpu").to(torch.float32))
    with pytest.raises(ValueError):
        pipeline.DESeq(d["counts"], x, sizeFactors=d["sizeFactors"], engine=emu_dev, weights=np.ones((30, 11)))
    for kw in ({"betaPrior": True, "factors": [np.r_[np.zeros(6), np.ones(6)].astype(int)]},
               {"minReplicatesForReplace": 7}):
        with pytest.raises(ValueError):
            DP.DESeq_device(y, x, d["sizeFactors"], weights=gm64(ok, "cpu"), **kw)
        with pytest.raises(ValueError):
            pipeline.DESeq(d["counts"], x, sizeFactors=d["sizeFactors"], engine=emu_dev, weights=ok, **kw)
    w = np.ones((30, 12))
    w[2, 1] = -1.0
    with pytest.raises(ValueError):
        DP.getContrast_device(y, x, d["sizeFactors"], torch.full((30,), 0.1, dtype=torch.float64),
                              torch.zeros((30, 2), dtype=torch.float64), [0.0, 1.0], weights=gm64(w, "cpu"))


# ---------------------------------------------------------------- DESeq_device(weights) against pipeline.DESeq(weights)

def _zi_weights(n, m, seed, frac_low=0.3, low=None, counts=None):
    """zinbwave-like weights: most entries in (0.5, 1], a fraction near zero (1e-4 .. 1e-2; at the entries of `low`
    when given, e.g. the dropouts) or exactly zero.  With `counts`, every row keeps a positive weight on one of its
    non-zero counts: otherwise its weighted baseMean is 0 and the reference stops (NA rough-vs-moments estimate)."""
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.5, 1.0, (n, m))
    if low is None:
        low = rng.random((n, m)) < frac_low
    w[low] = 10.0 ** rng.uniform(-4, -2, int(low.sum()))
    w[rng.random((n, m)) < 0.05] = 0.0
    w[:, 0] = 1.0
    if counts is not None:
        dead = (counts.sum(axis=1) > 0) & ((w * counts).sum(axis=1) == 0)
        w[dead, np.argmax(counts[dead], axis=1)] = 1.0
    return w


def _fail_some_rows(w, x):
    """Row 2 (and row 1 for factor designs) gets weights that leave the design rank deficient: weight only on the
    samples where the last column takes its maximum (row 1: zero weight there)."""
    w = w.copy()
    col = x[:, -1] == x[:, -1].max()
    w[1, col] = 0.0
    w[2, ~col] = 0.0
    w[2, col] = np.maximum(w[2, col], 0.5)
    return w


def _compare_weighted(engine, oracle, counts, x, sf, w, dev, minmu=0.5, tol=1e-6):
    """The acceptance rule of test_device_pipeline_matches_host_pipeline: every gene whose two dispersion line
    searches took the same number of steps on both sides agrees within 1e-6; the others must be rare and
    oracle-certified knife edges (decision margin below 4096 rounding bounds)."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        host = pipeline.DESeq(counts, x, sizeFactors=sf, engine=engine, useOptim=False, weights=w, minmu=minmu)
        dv = DP.DESeq_device(gm64(counts, dev), x, sf, useOptim=False, weights=gm64(w, dev), minmu=minmu)
    idx = dv["idx"].cpu().numpy()
    assert np.array_equal(idx, host["idx"])
    assert np.array_equal(dv["weightsFail"].cpu().numpy(), host["weightsFail"])
    m = x.shape[0]
    assert np.array_equal(dv["weights"].cpu().numpy()[:, :m], host["weights"])
    assert np.max(rel_err(dv["baseMean"].cpu().numpy(), host["baseMean"][idx])) < 1e-12
    same = ((dv["dispGeneIter"].cpu().numpy() == host["dispGeneIter"][idx])
            & (dv["dispIter"].cpu().numpy() == host["dispIter"][idx]))
    if np.any(~same):
        from test_device_pipeline_gpu import _MarginOracle
        assert np.mean(~same) <= 0.01
        mo = _MarginOracle(oracle)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            pipeline.DESeq(counts, x, sizeFactors=sf, engine=mo, useOptim=False, weights=w, minmu=minmu)
        margin = np.minimum(mo.margins[-2], mo.margins[-1])
        assert np.all(margin[~same] < 4096), (np.flatnonzero(~same)[:8], margin[~same][:8])
    for k in ("dispGeneEst", "dispMAP", "dispersion"):
        assert np.max(rel_err(dv[k].cpu().numpy()[same], host[k][idx][same])) < tol, k
    conv = (host["betaConv"][idx] == 1) & same
    it_same = dv["betaIter"].cpu().numpy()[conv] == host["betaIter"][idx][conv]
    assert np.mean(it_same) > 0.995
    for k in ("betaMatrix", "betaSE", "WaldStatistic", "deviance"):
        floor = 1e-6 if k != "deviance" else 1e-12
        e = rel_err(dv[k].cpu().numpy()[conv], host[k][idx][conv], floor=floor)
        assert np.max(e) < tol, (k, np.max(e))
    assert np.max(np.abs(dv["WaldPvalue"].cpu().numpy()[conv] - host["WaldPvalue"][idx][conv])) < tol
    return host, dv


_PIPE_DESIGNS = {"condition12": lambda: __import__("deseq2_b200.synth").synth.design_condition(12),
                 "batch_condition36": lambda: __import__("deseq2_b200.synth").synth.design_batch_condition(36, 3),
                 "factor6_40": lambda: __import__("deseq2_b200.synth").synth.design_factor(40, 6),
                 "continuous40": lambda: np.c_[np.ones(40), np.linspace(-1.0, 1.0, 40)]}


@pytest.mark.parametrize("design", sorted(_PIPE_DESIGNS))
def test_device_pipeline_weights_match_host(emu_dev, oracle, design):
    x = _PIPE_DESIGNS[design]()
    n, m = 240, x.shape[0]
    d = _make(n, x, 13)
    counts = d["counts"].copy()
    counts[5] = 0
    w = _fail_some_rows(_zi_weights(n, m, 17, counts=counts), x)
    host, dv = _compare_weighted(emu_dev, oracle, counts, x, d["sizeFactors"], w, "cpu")
    assert host["weightsFail"][2] and (host["weightsFail"][1] or design == "continuous40")
    assert 5 not in dv["idx"].cpu().numpy() and 2 not in dv["idx"].cpu().numpy()


# ---------------------------------------------------------------- properties from the reference's test_weights.R

def _drop_sample_case(x, seed=21, n=150):
    d = _make(n, x, seed)
    keep = np.ones(x.shape[0], bool)
    keep[3] = False
    w = np.ones(d["counts"].shape)
    w[:, 3] = 0.0
    return d, keep, w


@pytest.mark.parametrize("reduced", ["condition", "intercept"])
def test_zero_weight_equals_dropping_the_sample_lrt(emu_dev, reduced):
    from deseq2_b200 import device_pipeline as DP, synth
    m = 14
    x = synth.design_batch_condition(m, 2) if reduced == "condition" else synth.design_condition(m)
    xr = x[:, [0, x.shape[1] - 1]] if reduced == "condition" else np.ones((m, 1))
    d, keep, w = _drop_sample_case(x)
    counts = d["counts"][d["counts"].sum(axis=1) > 0]
    w = w[: len(counts)]
    disp = torch.full((len(counts),), 0.2, dtype=torch.float64)
    # both IRLS runs to a tight deviance tolerance: with the default 1e-8 the two starts (beta0 is unweighted and
    # sees the zero-weight sample) leave differences of order sqrt(1e-8) in beta
    kw = dict(useOptim=False, betaTol=1e-13, maxit=500)
    a = DP.nbinomLRT_device(gm64(counts, "cpu"), x, xr, d["sizeFactors"], disp, weights=gm64(w, "cpu"), **kw)
    yk = gm64(counts[:, keep], "cpu")
    # an intercept-only reduced model takes R's closed form only with weights (the unweighted device LRT fits it by
    # IRLS): all-ones weights on the dropped-sample run give the unweighted closed form
    wk = torch.ones_like(yk) if reduced == "intercept" else None
    b = DP.nbinomLRT_device(yk, x[keep], xr[keep], d["sizeFactors"][keep], disp, weights=wk, **kw)
    for k in ("betaMatrix", "betaSE", "deviance", "LRTStatistic"):
        e = rel_err(a[k].cpu().numpy(), b[k].cpu().numpy(), floor=1.0)
        assert np.max(e) < 1e-6, (k, np.max(e))
    assert torch.all(a["H"][:, 3] == 0.0)


def test_zero_weight_equals_dropping_the_sample_dispersion(emu_dev):
    """dispGeneEst with a zero weight on one sample against the run without it, within R's tolerance 1e-3 (the
    weighted run starts from other moments and clamps the weight at 1e-6).  Unit
    size factors as in the reference's test: then the weighted GLM mean equals the unweighted run's linear mu."""
    from deseq2_b200 import device_pipeline as DP, synth
    x = synth.design_condition(12)
    d, keep, w = _drop_sample_case(x, seed=5, n=300)
    counts, sf = d["counts"], np.ones(12)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        # the weighted run's mu is an IRLS fit (no linear mu with weights): to a tight tolerance it is the group mean
        a = DP.DESeq_device(gm64(counts, "cpu"), x, sf, weights=gm64(w, "cpu"), betaTol=1e-12, dispTol=1e-12)
        b = DP.DESeq_device(gm64(counts[:, keep], "cpu"), x[keep], sf[keep], betaTol=1e-12, dispTol=1e-12)
    ia, ib = a["idx"].cpu().numpy(), b["idx"].cpu().numpy()
    common = np.intersect1d(ia, ib)
    ga = a["dispGeneEst"].cpu().numpy()[np.searchsorted(ia, common)]
    gb = b["dispGeneEst"].cpu().numpy()[np.searchsorted(ib, common)]
    # genes where either run fell back to its start value (the noIncrease rule, R/core.R:806-808: the log posterior
    # rose by less than 1e-6 relative) are left out: the starts differ by design, the weighted moments average over
    # all m samples
    a0a = DP.prep(gm64(counts, "cpu"), x, sf, want_mu=False, weights=gm64(w, "cpu"))["alpha0"].cpu().numpy()[ia]
    a0b = DP.prep(gm64(counts[:, keep], "cpu"), x[keep], sf[keep], want_mu=False)["alpha0"].cpu().numpy()
    fallback = (ga == a0a[np.searchsorted(ia, common)]) | (gb == a0b[ib][np.searchsorted(ib, common)])
    fallback |= (ga == 12.0) | (gb == 11.0)             # at the upper bound max(10, m), which differs by one sample
    assert np.mean(fallback) < 0.2
    e = rel_err(ga, gb)[~fallback]
    assert np.mean(e < 1e-3) >= 0.99, np.sort(e)[-5:]  # the rest: a grid refit on one side only


def test_downweighting_an_outlier_lowers_dispersion(emu_dev):
    from deseq2_b200 import device_pipeline as DP, synth
    x = synth.design_condition(12)
    d = _make(200, x, 6)
    counts = d["counts"].copy()
    counts[0] = np.maximum(counts[0], 20)
    counts[0, 0] = 100 * counts[0].max()
    w = np.ones(counts.shape)
    w[0, 0] = 0.0
    y = gm64(counts, "cpu")
    plain = DP.DESeq_device(y, x, np.ones(12))
    weighted = DP.DESeq_device(y, x, np.ones(12), weights=gm64(w, "cpu"))
    assert weighted["dispMAP"][0] < plain["dispMAP"][0]
    assert weighted["dispGeneEst"][0] < plain["dispGeneEst"][0]


def test_get_contrast_weights_matches_host(emu_dev):
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = synth.design_batch_condition(36, 3)
    d = _make(200, x, 31)
    w = _fail_some_rows(_zi_weights(200, 36, 3, counts=d["counts"]), x)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        dv = DP.DESeq_device(gm64(d["counts"], "cpu"), x, d["sizeFactors"], weights=gm64(w, "cpu"), useOptim=False)
    idx = dv["idx"].cpu().numpy()
    counts = d["counts"][idx]
    ynz = gm64(counts, "cpu")
    nf = np.broadcast_to(d["sizeFactors"][None, :], counts.shape)
    disp, beta = dv["dispersion"].cpu().numpy(), dv["betaMatrix"].cpu().numpy()
    for con in ([0, 1, -1, 0], [0, 0, 0, 1], [0, 0.5, 0.5, -1]):
        for wd in (dv["weights"], gm64(w[idx], "cpu")):           # normalised or raw: the same normalisation
            g = DP.getContrast_device(ynz, x, d["sizeFactors"], dv["dispersion"], dv["betaMatrix"], con, weights=wd)
            h = pipeline.getContrast(counts, nf, x, disp, beta, con, engine=emu_dev, weights=w[idx])
            for k in ("log2FoldChange", "lfcSE", "stat"):
                assert np.max(rel_err(g[k].cpu().numpy(), h[k], floor=1e-6)) < 1e-6, k
            assert np.max(np.abs(g["pvalue"].cpu().numpy() - h["pvalue"])) < 1e-6


# ---------------------------------------------------------------- sharding

def _sharded_data(n, m):
    from deseq2_b200 import synth
    x = synth.design_batch_condition(m, 3)
    d = synth.make_example_counts(n, m, x=x, seed=91)
    return d["counts"], x, d["sizeFactors"], _fail_some_rows(_zi_weights(n, m, 5), x)


def _sharded_rank(rank, world, dev, n, m):
    from deseq2_b200 import sharded
    K, x, sf, w = _sharded_data(n, m)
    lo, hi = sharded.shard_bounds(n, world, rank)
    y = gm(K[lo:hi], dev)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        plain = sharded.sharded_DESeq_device(y, x, sf)
        r = sharded.sharded_DESeq_device(y, x, sf, weights=gm(w[lo:hi], dev))
    return {"gathered": r["gathered"], "extra_collectives": r["collectives"] - plain["collectives"],
            "n_local": r["idx"].numel()}


def _check_sharded(backend, n, m, world=2):
    """Weights sharded by rows: every gathered result equals the single-process run bit for bit, through the same
    collectives as the unweighted run (the trend step's gather carries the weighted baseMean)."""
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_sharded_rank, n, m, world=world, backend=backend)
    K, x, sf, w = _sharded_data(n, m)
    dev = DEVICE[backend]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        whole = DP.DESeq_device(gm64(K, dev), x, sf, weights=gm64(w, dev))
    assert bool(whole["weightsFail"].any())
    for g in got:
        assert 0 < g["n_local"] < whole["idx"].numel()
        assert g["extra_collectives"] == 0
        for k in ("dispersion", "betaMatrix", "betaSE", "WaldPvalue"):
            assert np.array_equal(g["gathered"][k], whole[k].cpu().numpy(), equal_nan=True), k


def test_sharded_weights_equal_whole(emu_dev):
    _check_sharded("gloo", 400, 12)


# ---------------------------------------------------------------- GPU (or the emulator with B200NB_LIB)

@pytest.mark.gpu
@pytest.mark.parametrize("design,n,m,poscounts", [("condition", 2000, 100, False), ("batch", 3000, 36, False),
                                                  ("factor10", 600, 420, False), ("condition", 2000, 1000, True)])
def test_device_pipeline_weights_match_host_gpu(engine, oracle, design, n, m, poscounts):
    """Long rows (m = 420, 1000) with weights leave the segmented general-p kernels; the last case is the
    single-cell setting: zero-inflated weights, poscounts size factors, minmu = 1e-6."""
    from deseq2_b200 import device_pipeline as DP, synth
    x = {"condition": synth.design_condition, "batch": lambda k: synth.design_batch_condition(k, 3),
         "factor10": lambda k: synth.design_factor(k, 10)}[design](m)
    d = _make(n, x, 11)
    counts = d["counts"].copy()
    counts[7] = 0
    sf = d["sizeFactors"]
    minmu = 0.5
    low = None
    if poscounts:
        low = np.random.default_rng(2).random(counts.shape) < 0.3
        counts[low] = 0                                                # dropouts, down-weighted
        sf = DP.size_factors(gm64(counts, DEV), m, type="poscounts")["sizeFactors"].cpu().numpy()
        minmu = 1e-6
    w = _fail_some_rows(_zi_weights(n, m, 19, low=low, counts=counts), x)
    _compare_weighted(engine, oracle, counts, x, sf, w, DEV, minmu=minmu)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C2", "C4"])
def test_config_sizes_with_weights(engine, config):
    """BASELINE C2 (50 000 x 100, ~condition) and C4 (50 000 x 1000, 10-level factor) with weights."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    m = 100 if config == "C2" else 1000
    n = 50000 if DEV == "cuda" else 1000
    x = synth.design_condition(m) if config == "C2" else synth.design_factor(m, 10)
    d = synth.make_example_counts(n, m, x=x, seed=4)
    w = _fail_some_rows(_zi_weights(n, m, 23, counts=d["counts"]), x)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        dv = DP.DESeq_device(gm64(d["counts"], DEV), x, d["sizeFactors"], weights=gm64(w, DEV))
    for k in ("dispersion", "betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue", "deviance"):
        assert torch.isfinite(dv[k]).all(), k
    assert (dv["betaIter"] < 100).double().mean().item() >= 0.99
    sample = np.sort(np.random.default_rng(0).choice(n, min(n, 2000), replace=False))
    sample[:2] = [1, 2]
    _, fail = pipeline.getAndCheckWeights(w[sample], x)
    assert np.array_equal(dv["weightsFail"].cpu().numpy()[sample], fail)
    assert fail[1]


@pytest.mark.gpu
def test_sharded_weights_over_nccl_equals_whole(engine):
    _check_sharded("nccl", 20000, 60, nccl_world())
