"""DESeq(sfType = "iterate") and fitType = "mean" on the device: the objective kernels (b200nb_sf_iterate_objective_dev,
csrc/sf_iterate.cuh) against the direct numpy evaluation pipeline.iterateObjective, size_factors_iterate against the
host mirror pipeline.estimateSizeFactorsIterate driving the oracle engine, the reference's test_size_factor.R property,
the error cases, and DESeq_device(fitType = "mean") against pipeline.DESeq, including a two-rank gloo run.
The CPU tests run the engine's CUDA source on the SIMT emulator (`emu` fixture); the `-m gpu` tests run on a GPU, or on
the emulator when B200NB_LIB points at it."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm, gm64, rel_err
from ranks import DEVICE, nccl_world, run_ranks


def _objective_case(n, m, seed, ties=False):
    """Zero-heavy rows, random q, dispersions and log size factors.  ties: n // 10 + 2 identical rows (counts, q and
    dispersion) whose log-likelihood is the lowest in every column, so the quantile's order statistics are copies of
    one value."""
    rng = np.random.default_rng(seed)
    K = rng.negative_binomial(2, 0.15, (n, m)).astype(np.float64)
    K[: n // 3, : max(1, m // 2)] = 0.0
    q = np.exp(rng.normal(1.0, 1.0, (n, m)))
    alpha = np.exp(rng.normal(-2.0, 1.0, n))
    par = rng.normal(0.0, 0.3, m)
    if ties:
        b = n // 10 + 2
        K[-b:], q[-b:], alpha[-b:] = 400.0, 1.0, 0.01
    return K, q, alpha, par


def _sorted_center_ll(K, q, alpha, par):
    from deseq2_b200 import pipeline
    return np.sort(pipeline.nbinomLogLike(K, q * np.exp(par - np.mean(par))[None, :], alpha))


def _device_objective(K, q, alpha, par, dev, f64=True, tile=0):
    from deseq2_b200 import device as D, device_pipeline as DP
    y = D.to_gene_major(np.asarray(K, dtype=np.float64 if f64 else np.int32), torch.device(dev))
    return DP.sf_iterate_objective(y, gm64(q, dev), torch.as_tensor(alpha, device=dev),
                                   torch.as_tensor(np.asarray(par, dtype=np.float64), device=dev), len(par),
                                   max_tile_cols=tile).cpu().numpy()


def _objective_err(got, want):
    return np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-300))


# ---------------------------------------------------------------- the objective kernels

@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("n,m,tile", [(1, 2, 0), (21, 3, 2), (401, 5, 3), (1000, 2, 0), (2500, 100, 64),
                                      (300, 100, 0)])
def test_objective_matches_direct(emu_dev, f64, n, m, tile, ties):
    """Every one of the 2m + 1 values within 1e-12 of the direct evaluation; n = 21 and 401 make (n - 1) Q an
    exact integer; tile > 0 splits the columns into several tiles; m = 3, 5 leave ld padding.  With ties the two
    order statistics of the quantile are copies of one value (at n = 1000, 2500, 300 the index is fractional, so the
    kernel's x[hi] = x[lo] branch decides) and every copy is left out of the sum."""
    from deseq2_b200 import pipeline
    K, q, alpha, par = _objective_case(n, m, n + m, ties=ties and n > 1)
    if ties and n > 1:
        x = _sorted_center_ll(K, q, alpha, par)
        lo = int(np.floor((n - 1) * 0.05))
        assert x[lo] == x[min(lo + 1, n - 1)] == x[0]
    want = pipeline.iterateObjective(K, q, alpha, par)
    got = _device_objective(K, q, alpha, par, "cpu", f64=f64, tile=tile)
    assert got.shape == (2 * m + 1,)
    if n == 1:
        assert np.all(got == 0.0) and np.all(want == 0.0)     # nothing lies strictly above the only value
    else:
        assert _objective_err(got, want) < 1e-12
    again = _device_objective(K, q, alpha, par, "cpu", f64=f64, tile=tile)
    assert np.array_equal(got.view(np.int64), again.view(np.int64))


@pytest.mark.parametrize("n", [21, 401])
def test_objective_exact_integer_quantile_index(emu_dev, n):
    """(n - 1) Q is an exact integer: the quantile is the order statistic x[1 + (n - 1) Q] itself, no interpolation;
    fn(par) is the sum of the values strictly above it, computed here from the sorted log-likelihoods."""
    K, q, alpha, par = _objective_case(n, 4, 3 * n)
    assert float((n - 1) * 0.05).is_integer()
    x = _sorted_center_ll(K, q, alpha, par)
    qs = x[int((n - 1) * 0.05)]
    want = x[x > qs].sum()
    got = _device_objective(K, q, alpha, par, "cpu")[0]
    assert abs(got - want) < 1e-12 * abs(want)
    assert np.sum(x > qs) == n - 1 - int((n - 1) * 0.05)


def test_objective_abi_rejects_bad_arguments(emu_dev):
    from deseq2_b200 import _lib
    L = _lib.lib()
    K, q, alpha, par = _objective_case(10, 3, 1)
    y, qd = gm64(K, "cpu"), gm64(q, "cpu")
    a, pd = torch.as_tensor(alpha), torch.as_tensor(par)
    out = torch.empty(7, dtype=torch.float64)
    P = lambda t: C.c_void_p(t.data_ptr())
    good = dict(y=P(y), q=P(qd), a=P(a), p=P(pd), h=1e-3, Q=0.05, n=10, m=3, ld=4, tile=0, out=P(out))

    def call(**kw):
        g = dict(good, **kw)
        return L.b200nb_sf_iterate_objective_dev(g["y"], 1, g["q"], g["a"], g["p"], g["h"], g["Q"], g["n"], g["m"],
                                                 g["ld"], g["tile"], g["out"], None)

    assert call() == 0
    for bad in (dict(n=0), dict(m=0), dict(h=0.0), dict(h=-1e-3), dict(h=float("nan")), dict(h=float("inf")),
                dict(Q=-0.1), dict(Q=1.0), dict(Q=float("nan")), dict(y=None), dict(q=None), dict(a=None),
                dict(p=None), dict(out=None), dict(ld=2), dict(tile=-1)):
        assert call(**bad) != 0, bad
        assert L.b200nb_last_error()


# ---------------------------------------------------------------- size_factors_iterate against the host mirror

def _reference_property_counts():
    """test_size_factor.R:20-45: true s = 2^(-2,-1,0,0,1,2) per pair of samples, dispersion 0.01, 100 genes, one zero
    per gene and a 10^6 outlier."""
    rng = np.random.default_rng(1)
    true_sf = 2.0 ** np.repeat([-2, -1, 0, 0, 1, 2], 2)
    n, m = 100, 12
    beta = rng.normal(np.log(50.0), 1.0, n)
    mu = np.exp(beta)[:, None] * true_sf[None, :]
    cts = rng.negative_binomial(1 / 0.01, (1 / 0.01) / (1 / 0.01 + mu)).astype(np.int64)
    cts[np.arange(n), rng.integers(0, m, n)] = 0
    cts[0, 0] = 1000000
    return cts, true_sf


def _check_lm(sf, true_sf):
    slope, intercept = np.polyfit(true_sf, sf, 1)
    assert abs(intercept) < 0.1 and abs(slope - 1.0) < 0.1, (intercept, slope)


def test_reference_property_host_and_device(emu_dev, oracle):
    from deseq2_b200 import device_pipeline as DP, pipeline
    cts, true_sf = _reference_property_counts()
    host = pipeline.estimateSizeFactorsIterate(cts, engine=oracle)
    _check_lm(host["sizeFactors"], true_sf)
    dv = DP.size_factors_iterate(gm64(cts, "cpu"), 12)
    _check_lm(dv["sizeFactors"], true_sf)
    assert dv["iterations"] == host["iterations"]
    assert np.max(rel_err(dv["sizeFactors"], host["sizeFactors"])) < 1e-4


def _compare_iterate(oracle, counts, dev, **kw):
    """Equal outer iteration counts, size factors within 1e-4 (factr = 1e7's resolution on these objectives: the
    evaluators agree to 1e-12, so the two optimiser runs differ only through the last bits of the objective),
    last-iteration dispersions within 1e-6."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    m = counts.shape[1]
    host = pipeline.estimateSizeFactorsIterate(counts, engine=oracle)
    dv = DP.size_factors_iterate(gm64(counts, dev), m, **kw)
    assert dv["iterations"] == host["iterations"]
    assert np.max(rel_err(dv["sizeFactors"], host["sizeFactors"])) < 1e-4
    assert np.max(rel_err(dv["dispersion"].cpu().numpy(), host["last"]["dispersion"])) < 1e-6
    assert len(dv["evaluations"]) == dv["iterations"]
    return host, dv


def test_size_factors_iterate_matches_host(emu_dev, oracle):
    from deseq2_b200 import synth
    d = synth.make_example_counts(300, 12, x=synth.design_condition(12), seed=21)
    counts = d["counts"].copy()
    counts[np.arange(300), np.arange(300) % 12] = 0                  # every gene has a zero: "ratio" cannot run
    counts[3] = 0
    _compare_iterate(oracle, counts, "cpu", max_tile_cols=7)


def test_replay_host_optimizer_points(emu_dev, oracle, monkeypatch):
    """The device objective at every point the host mirror's optimiser visited, with the host's q and dispersions."""
    from deseq2_b200 import pipeline, synth
    d = synth.make_example_counts(200, 6, x=synth.design_condition(6), seed=5)
    counts = d["counts"].copy()
    counts[np.arange(200), np.arange(200) % 6] = 0
    seen = []
    real = pipeline.iterateObjective

    def spy(counts_, q, disps, par, h=1e-3, Q=0.05):
        v = real(counts_, q, disps, par, h, Q)
        seen.append((counts_, q, disps, np.array(par), v))
        return v

    monkeypatch.setattr(pipeline, "iterateObjective", spy)
    pipeline.estimateSizeFactorsIterate(counts, engine=oracle)
    assert len(seen) > 5
    for cts, q, disps, par, want in seen:
        got = _device_objective(cts, q, disps, par, "cpu")
        assert _objective_err(got, want) < 1e-12


# ---------------------------------------------------------------- errors

def test_iterate_errors(emu_dev, oracle):
    from deseq2_b200 import device_pipeline as DP, pipeline, sharded
    cts, _ = _reference_property_counts()
    y = gm64(cts, "cpu")
    with pytest.raises(ValueError, match="did not converge"):
        DP.size_factors_iterate(y, 12, niter=1)
    with pytest.raises(ValueError, match="did not converge"):
        pipeline.estimateSizeFactorsIterate(cts, niter=1, engine=oracle)
    x = np.ones((12, 1))
    ones = gm64(np.ones(cts.shape), "cpu")
    for kw in (dict(weights=ones), dict(normalizationFactors=ones), dict(avgTxLength=ones)):
        with pytest.raises(ValueError, match="iterate"):
            DP.DESeq_device(y, x, sfType="iterate", **kw)
    with pytest.raises(ValueError, match="iterate"):
        pipeline.DESeq(cts, x, sfType="iterate", weights=np.ones(cts.shape), engine=oracle)
    with pytest.raises(ValueError, match="sizeFactors"):
        sharded.sharded_DESeq_device(y, x, sfType="iterate")
    with pytest.raises(ValueError, match="sfType"):
        DP.DESeq_device(y, x, sfType="median")
    with pytest.raises(ValueError, match="fitType"):
        DP.DESeq_device(y, x, fitType="local")
    # every gene-wise estimate below 100 minDisp: R's stop in estimateDispersionsFit
    pois = np.random.default_rng(3).poisson(np.repeat([[5.0, 20.0, 80.0]], 60, axis=0).repeat(4, axis=1))
    with pytest.raises(ValueError, match="within 2 orders of magnitude"):
        DP.size_factors_iterate(gm64(pois, "cpu"), 12, minDisp=1.0)
    with pytest.raises(ValueError, match="within 2 orders of magnitude"):
        pipeline.estimateSizeFactorsIterate(pois, engine=oracle, minDisp=1.0)


# ---------------------------------------------------------------- fitType = "mean"

def _design(name):
    from deseq2_b200 import synth
    return {"condition12": lambda: synth.design_condition(12),
            "batch_condition36": lambda: synth.design_batch_condition(36, 3),
            "factor6_40": lambda: synth.design_factor(40, 6),
            "continuous40": lambda: np.c_[np.ones(40), np.linspace(-1.0, 1.0, 40)]}[name]()


def _compare_mean(oracle, counts, x, dev, tol=1e-6, fitType="mean", **kw):
    """test_norm_factors_device's acceptance rule: genes whose two dispersion line searches took the same number of
    steps on both sides agree within tol; the others must be rare."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    host = pipeline.DESeq(counts, x, engine=oracle, useOptim=False, fitType=fitType, **kw)
    dv = DP.DESeq_device(gm64(counts, dev), x, useOptim=False, fitType=fitType, **kw)
    idx = dv["idx"].cpu().numpy()
    assert dv["fitType"] == host["fitType"] == fitType
    if fitType == "mean":
        assert "trendCoefs" not in dv and "trendCoefs" not in host
        assert abs(dv["meanDisp"] - host["meanDisp"]) < tol * host["meanDisp"]
    else:
        assert np.max(rel_err(dv["trendCoefs"].cpu().numpy(), host["trendCoefs"])) < tol
    assert np.max(rel_err(dv["dispFit"].cpu().numpy(), host["dispFit"][idx])) < tol
    same = ((dv["dispGeneIter"].cpu().numpy() == host["dispGeneIter"][idx])
            & (dv["dispIter"].cpu().numpy() == host["dispIter"][idx]))
    assert np.mean(~same) <= 0.02
    for k in ("dispGeneEst", "dispMAP", "dispersion"):
        assert np.max(rel_err(dv[k].cpu().numpy()[same], host[k][idx][same])) < tol, k
    conv = (host["betaConv"][idx] == 1) & same
    for k in ("betaMatrix", "betaSE", "WaldStatistic"):
        assert np.max(rel_err(dv[k].cpu().numpy()[conv], host[k][idx][conv], floor=1e-6)) < tol, k
    return host, dv


@pytest.mark.parametrize("design", ["condition12", "batch_condition36", "factor6_40", "continuous40"])
def test_device_pipeline_mean_matches_host(emu_dev, oracle, design):
    from deseq2_b200 import synth
    x = _design(design)
    d = synth.make_example_counts(240, x.shape[0], x=x, seed=31, betaSD=0.3)
    counts = d["counts"].copy()
    counts[5] = 0
    _compare_mean(oracle, counts, x, "cpu", sizeFactors=d["sizeFactors"])


def test_device_pipeline_mean_with_replacement_and_iterate(emu_dev, oracle):
    from deseq2_b200 import synth
    # batch x condition at 48 samples: 8 per cell, so every sample is replaceable, and the gene-wise mean of the refit
    # comes from a GLM fit (fewer coefficients than design groups)
    for x in (synth.design_batch_condition(48, 3), synth.design_condition(16)):
        d = synth.make_example_counts(240, x.shape[0], x=x, seed=33, betaSD=0.3)
        counts = d["counts"].copy()
        counts[[10, 20, 30, 40], [1, 2, 9, 12]] = 40 * counts[[10, 20, 30, 40]].max(axis=1) + 200
        host, dv = _compare_mean(oracle, counts, x, "cpu", minReplicatesForReplace=7, sizeFactors=d["sizeFactors"])
        assert dv["n_replaced"] == int(host["replace"].sum()) > 0
    host, dv = _compare_mean(oracle, counts, x, "cpu", sfType="iterate")
    assert np.max(rel_err(dv["sizeFactors"], host["sizeFactors"])) < 1e-4
    assert dv["sfIterate"]["iterations"] == host["sfIterate"]["iterations"]


def test_iterate_size_factors_ignore_the_fit_minmu(emu_dev, oracle):
    """DESeq() hands minmu to the dispersion and Wald fits only: the iterate estimator runs its own estimateDispersions
    with minmu = 0.5 (R/core.R:388, 2596).  At minmu = 1e-6 (the single-cell setting) the device size factors are the
    bits of size_factors_iterate with its defaults, and the whole analysis matches pipeline.DESeq."""
    from deseq2_b200 import device_pipeline as DP, synth
    x = synth.design_condition(12)
    d = synth.make_example_counts(240, 12, x=x, seed=35, betaSD=0.3)
    counts = d["counts"].copy()
    counts[np.arange(240), np.arange(240) % 12] = 0                  # every gene has a zero
    host, dv = _compare_mean(oracle, counts, x, "cpu", fitType="parametric", sfType="iterate", minmu=1e-6)
    alone = DP.size_factors_iterate(gm64(counts, "cpu"), 12)["sizeFactors"]
    assert np.array_equal(dv["sizeFactors"], alone)
    assert np.max(rel_err(dv["sizeFactors"], host["sizeFactors"])) < 1e-4
    assert dv["sfIterate"]["iterations"] == host["sfIterate"]["iterations"]


def test_poscounts_size_factors_match_host(emu_dev, oracle):
    """sfType = "poscounts": the device estimate (geoMeanNZ, incoming-geoMeans rescaling) against
    pipeline.estimateSizeFactorsForMatrix(type = "poscounts"), alone and through DESeq()."""
    from deseq2_b200 import pipeline, synth
    x = synth.design_condition(12)
    d = synth.make_example_counts(240, 12, x=x, seed=37, betaSD=0.3)
    counts = d["counts"].copy()
    counts[np.arange(240), np.arange(240) % 12] = 0                  # "ratio" would have no usable gene
    counts[7] = 0
    sf = pipeline.estimateSizeFactorsForMatrix(counts, type="poscounts")
    assert abs(np.exp(np.mean(np.log(sf))) - 1.0) < 1e-14
    host, dv = _compare_mean(oracle, counts, x, "cpu", fitType="parametric", sfType="poscounts")
    assert np.array_equal(host["sizeFactors"], sf)
    assert np.max(rel_err(dv["sizeFactors"], sf)) < 1e-12


def test_mean_disp_trims(emu_dev):
    """n >= 1000: floor(n 0.001) order statistics leave at each end, as mean(trim = 0.001) does."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    rng = np.random.default_rng(4)
    d = np.exp(rng.normal(-2.0, 0.5, 2500))
    d[:2] = 1e3                                                      # would move an untrimmed mean by ~0.8
    d[3] = 1e-9                                                      # below 10 minDisp: not used
    want = pipeline.meanDispersionFit(d)
    kept = np.sort(d[d > 1e-7])
    assert abs(want - kept[2:-2].mean()) < 1e-14 * want             # floor(2499 * 0.001) = 2 from each end
    assert abs(want - kept.mean()) > 0.5
    got = float(DP.mean_disp(torch.as_tensor(d)).item())
    assert abs(got - want) < 1e-14 * want


def _sharded_data(n, m):
    from deseq2_b200 import synth
    x = synth.design_batch_condition(m, 3)
    d = synth.make_example_counts(n, m, x=x, seed=91)
    return d["counts"], x, d["sizeFactors"]


def _sharded_rank(rank, world, dev, n, m):
    from deseq2_b200 import sharded
    K, x, sf = _sharded_data(n, m)
    lo, hi = sharded.shard_bounds(n, world, rank)
    y = gm(K[lo:hi], dev)
    warnings.simplefilter("ignore")
    plain = sharded.sharded_DESeq_device(y, x, sf)
    r = sharded.sharded_DESeq_device(y, x, sf, fitType="mean")
    return {"gathered": r["gathered"], "extra_collectives": r["collectives"] - plain["collectives"],
            "meanDisp": r["meanDisp"]}


def _check_sharded(backend, n, m, world=2):
    """The same bits as one process (the trimmed mean is of the gathered estimates, in rank order = gene order) and
    the same number of collectives as the parametric run."""
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_sharded_rank, n, m, world=world, backend=backend)
    K, x, sf = _sharded_data(n, m)
    whole = DP.DESeq_device(gm64(K, DEVICE[backend]), x, sf, fitType="mean")
    for g in got:
        assert g["meanDisp"] == whole["meanDisp"]
        assert g["extra_collectives"] == 0
        for k in ("dispersion", "betaMatrix", "betaSE", "WaldPvalue"):
            assert np.array_equal(g["gathered"][k], whole[k].cpu().numpy()), k


def test_sharded_mean_equal_whole(emu_dev):
    _check_sharded("gloo", 400, 12)


# ---------------------------------------------------------------- GPU (or the emulator with B200NB_LIB)

@pytest.mark.gpu
@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("n,m,tile", [(21, 3, 0), (3001, 5, 4), (2000, 100, 0), (2000, 100, 37), (401, 2, 0)])
def test_objective_matches_direct_gpu(engine, f64, n, m, tile, ties):
    from deseq2_b200 import pipeline
    K, q, alpha, par = _objective_case(n, m, 7 * n + m, ties=ties)
    want = pipeline.iterateObjective(K, q, alpha, par)
    got = _device_objective(K, q, alpha, par, DEV, f64=f64, tile=tile)
    assert _objective_err(got, want) < 1e-12
    again = _device_objective(K, q, alpha, par, DEV, f64=f64, tile=tile)
    assert np.array_equal(got.view(np.int64), again.view(np.int64))


@pytest.mark.gpu
@pytest.mark.parametrize("n,m", [(2000, 12), (500, 40)])
def test_size_factors_iterate_matches_host_gpu(engine, oracle, n, m):
    from deseq2_b200 import synth
    d = synth.make_example_counts(n, m, x=synth.design_condition(m), seed=n + m)
    counts = d["counts"].copy()
    counts[np.arange(n), np.arange(n) % m] = 0
    _compare_iterate(oracle, counts, DEV)


@pytest.mark.gpu
def test_reference_property_gpu(engine):
    from deseq2_b200 import device_pipeline as DP
    cts, true_sf = _reference_property_counts()
    _check_lm(DP.size_factors_iterate(gm64(cts, DEV), 12)["sizeFactors"], true_sf)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["C2", "single_cell"])
def test_iterate_at_scale(engine, shape):
    """DESeq_device(sfType = "iterate") at C2 (50 000 x 100) and a single-cell-like 20 000 x 2000 shape completes;
    the objective at the final size factors matches the direct evaluation on a random subset of columns."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    n, m = (50000, 100) if shape == "C2" else (20000, 2000)
    if DEV != "cuda":
        n, m = n // 100, m // 20                     # the emulator: 500 x 5, 200 x 100
    d = synth.make_example_counts(n, m, x=synth.design_condition(m), seed=17)
    y = gm64(d["counts"], DEV)
    dv = DP.DESeq_device(y, synth.design_condition(m), sfType="iterate", fitType="mean")
    assert dv["sfIterate"]["iterations"] >= 2
    for k in ("dispersion", "betaMatrix", "WaldPvalue"):
        assert torch.isfinite(dv[k]).all(), k
    sf = dv["sizeFactors"]
    idx = dv["idx"]
    ynz = y[idx].contiguous()
    q, disp = dv["mu"][:, :m] / torch.as_tensor(sf, device=y.device)[None, :], dv["dispersion"]
    qd = torch.ones_like(dv["mu"])
    qd[:, :m] = q
    par = np.log(sf)
    got = DP.sf_iterate_objective(ynz, qd, disp.contiguous(), torch.as_tensor(par, device=y.device), m).cpu().numpy()
    cols = np.r_[0, np.random.default_rng(0).choice(np.arange(1, 2 * m + 1), 6, replace=False)]
    K = ynz[:, :m].cpu().numpy().astype(np.float64)
    qh, dh = q.cpu().numpy(), disp.cpu().numpy()
    want = np.empty(len(cols))
    for i, c in enumerate(cols):                  # iterateObjective's column c, evaluated alone
        p = par.copy()
        if c > 0:
            p[(c - 1) % m] += 1e-3 if c <= m else -1e-3
        ll = pipeline.nbinomLogLike(K, qh * np.exp(p - np.mean(p))[None, :], dh)
        want[i] = ll[ll > np.quantile(ll, 0.05, method="linear")].sum()
    assert _objective_err(got[cols], want) < 1e-12


@pytest.mark.gpu
def test_sharded_mean_over_nccl_equals_whole(engine):
    _check_sharded("nccl", 20000, 12, nccl_world())
