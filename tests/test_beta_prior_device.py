"""DESeq(betaPrior=TRUE) on the device: the weighted-quantile prior-variance kernel (b200nb_beta_prior_quantile_dev,
csrc/beta_prior.cuh) against the host restatement of estimateBetaPriorVar (pipeline.py), the device pipeline's MAP fit
on the expanded matrix against pipeline.DESeq(betaPrior=True) driving the same engine, and the gene-sharded run.
The CPU tests run the engine's CUDA source on the SIMT emulator (`emu` fixture); the `-m gpu` tests run on a GPU, or on
the emulator when B200NB_LIB points at it."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm, rel_err
from ranks import DEVICE, nccl_world, run_ranks


def _factor(m, levels):
    return (np.arange(m) * levels) // m


def _bc_factors(m):
    return [np.arange(m) % 3, (np.arange(m) // 3) % 2]          # = synth.design_batch_condition(m, 3)


def _host_columns(betaMatrix, fidx):
    """The columns the host restatement takes quantiles of, in the kernel's order."""
    from deseq2_b200 import device_pipeline as DP
    a, b, _ = DP.beta_prior_columns(fidx)
    return [betaMatrix[:, i] - (0.0 if j < 0 else betaMatrix[:, j]) for i, j in zip(a, b)], a, b


def _host_q(x, w, prob=0.95):
    from deseq2_b200 import pipeline
    fin = np.abs(x) < 10
    if fin.sum() == 0:
        return np.nan
    return pipeline.wtd_quantile(np.abs(x[fin]), w[fin], prob)


def _host_expanded(betaMatrix, factors, baseMean, dispFit):
    from deseq2_b200 import pipeline
    _, names, fidx, _ = pipeline.factorDesign(factors)
    _, mean_by_factor = pipeline.estimateBetaPriorVar(betaMatrix, names, fidx, baseMean, dispFit)
    efidx = pipeline.factorDesign(factors, expanded=True)[2]
    return np.array([1e6 if f < 0 else mean_by_factor[int(f)] for f in efidx])


def _check_kernel_vs_host(betaMatrix, factors, baseMean, dispFit, dev="cpu"):
    from deseq2_b200 import device_pipeline as DP, pipeline
    _, _, fidx, _ = pipeline.factorDesign(factors)
    T = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    bt = T(betaMatrix.T)
    cols, a, b = _host_columns(betaMatrix, fidx)
    w = 1.0 / (1.0 / baseMean + dispFit)
    if len(baseMean) > 1:
        q = DP.beta_prior_quantile(bt, T(baseMean), T(dispFit), a, b, 0.95).cpu().numpy()
        ref = np.array([_host_q(x, w) for x in cols])
        assert np.array_equal(np.isnan(q), np.isnan(ref))
        ok = ~np.isnan(ref)
        assert np.all(rel_err(q[ok], ref[ok], floor=1e-300) <= 1e-12), (q, ref)
    pv = DP.estimate_beta_prior_var(bt.T, factors, T(baseMean), T(dispFit)).cpu().numpy()
    ref = _host_expanded(betaMatrix, factors, baseMean, dispFit)
    assert np.all(rel_err(pv, ref, floor=1e-300) <= 1e-12), (pv, ref)
    return pv


def _inputs(n, p, seed, sd=1.5):
    rng = np.random.default_rng(seed)
    beta = rng.normal(0.0, sd, (n, p))
    baseMean = np.exp(rng.normal(4.0, 2.0, n))
    dispFit = 0.05 + 2.0 / baseMean
    return beta, baseMean, dispFit


@pytest.mark.parametrize("n", [2, 3, 7, 40, 999, 20000])
def test_kernel_matches_host_random(emu_dev, n):
    factors = [_factor(max(n, 8), 4)]
    beta, bm, df = _inputs(n, 4, seed=n)
    _check_kernel_vs_host(beta, factors, bm, df)


@pytest.mark.parametrize("levels", [[2], [3], [4], [3, 2], [4, 3]])
def test_kernel_matches_host_designs(emu_dev, levels):
    m = 24
    factors = [_factor(m, L) if k == 0 else np.arange(m) % L for k, L in enumerate(levels)]
    p = 1 + sum(L - 1 for L in levels)
    beta, bm, df = _inputs(3000, p, seed=sum(levels))
    _check_kernel_vs_host(beta, factors, bm, df)


def test_kernel_heavy_ties(emu_dev):
    beta, bm, df = _inputs(5000, 4, seed=3, sd=0.3)
    _check_kernel_vs_host(np.round(beta, 2), [_factor(16, 4)], bm, df)


def test_kernel_nan_large_and_empty_columns(emu_dev):
    beta, bm, df = _inputs(2500, 4, seed=4)
    beta[::7, 1] = np.nan
    beta[::5, 2] = 12.0                         # |x| >= 10: not kept
    beta[3::11, 3] = -10.0
    beta[:, 3] = np.where(np.arange(2500) % 3 == 0, 25.0, beta[:, 3])
    pv = _check_kernel_vs_host(beta, [_factor(16, 4)], bm, df)
    assert np.all(np.isfinite(pv))
    # every entry of one column filtered: that column's variance is 1e6 (a 2-level factor has no contrast)
    beta2, bm2, df2 = _inputs(300, 3, seed=5)
    beta2[:, 2] = 11.0
    pv2 = _check_kernel_vs_host(beta2, [_factor(12, 2), np.arange(12) % 2], bm2, df2)
    assert pv2[-1] == 1e6 and pv2[-2] == 1e6


@pytest.mark.parametrize("n", [2, 5, 21, 100, 2000])
def test_kernel_constant_weights(emu_dev, n):
    """Equal weights put every cumulative weight on an integer: the order statistic is then decided by the slack
    v - 1e-12 max(1, v) of the host restatement."""
    beta, _, _ = _inputs(n, 4, seed=n + 100)
    _check_kernel_vs_host(beta, [_factor(16, 4)], np.full(n, 50.0), np.full(n, 0.1))


def test_single_gene_uses_squared_betas(emu_dev):
    beta, bm, df = _inputs(1, 4, seed=8)
    pv = _check_kernel_vs_host(beta, [_factor(16, 4)], bm, df)
    b = beta[0]
    sq = [b[1] ** 2, b[2] ** 2, b[3] ** 2, (b[2] - b[1]) ** 2, (b[3] - b[1]) ** 2, (b[3] - b[2]) ** 2]
    assert abs(pv[1] - np.mean(sq)) <= 1e-12 * pv[1]


def test_kernel_is_deterministic_and_checks_arguments(emu_dev):
    from deseq2_b200 import _lib, device_pipeline as DP
    beta, bm, df = _inputs(5000, 4, seed=9)
    bt, bmt, dft = (torch.as_tensor(np.ascontiguousarray(v)) for v in (beta.T, bm, df))
    a, b, _ = DP.beta_prior_columns(np.array([-1, 0, 0, 0]))
    q1 = DP.beta_prior_quantile(bt, bmt, dft, a, b, 0.95)
    q2 = DP.beta_prior_quantile(bt, bmt, dft, a, b, 0.95)
    assert torch.equal(q1, q2)
    L = _lib.lib()
    out = torch.empty(2, dtype=torch.float64)
    p_ = lambda t: C.c_void_p(t.data_ptr())
    ok_a, ok_b = torch.tensor([1, 2], dtype=torch.int32), torch.tensor([-1, 1], dtype=torch.int32)
    calls = {"n": (0, 4, ok_a, ok_b, 2, 0.95), "p": (100, 0, ok_a, ok_b, 2, 0.95), "k": (100, 4, ok_a, ok_b, -1, 0.95),
             "prob0": (100, 4, ok_a, ok_b, 2, 0.0), "prob1": (100, 4, ok_a, ok_b, 2, 1.0),
             "a": (100, 4, torch.tensor([1, 4], dtype=torch.int32), ok_b, 2, 0.95),
             "b": (100, 4, ok_a, torch.tensor([-2, 1], dtype=torch.int32), 2, 0.95),
             "b_hi": (100, 4, ok_a, torch.tensor([-1, 4], dtype=torch.int32), 2, 0.95)}
    for name, (n, p, ca, cb, k, prob) in calls.items():
        rc = L.b200nb_beta_prior_quantile_dev(p_(bt), n, p, p_(bmt), p_(dft), p_(ca), p_(cb), k, prob, p_(out),
                                              C.c_void_p(0))
        assert rc != 0, name
        assert L.b200nb_last_error().decode(), name
    rc = L.b200nb_beta_prior_quantile_dev(p_(bt), 100, 4, p_(bmt), p_(dft), p_(ok_a), p_(ok_b), 0, 0.95, p_(out),
                                          C.c_void_p(0))
    assert rc == 0


# ---------------------------------------------------------------- the pipeline with betaPrior=TRUE

def _compare_pipelines(engine, oracle, counts, x, factors, sizeFactors, dev, tol=1e-6):
    """The acceptance rule of test_device_pipeline_matches_host_pipeline, on the MAP results: every gene whose two
    line searches took the same number of steps on both sides agrees within 1e-6; the others must be rare."""
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline
    host = pipeline.DESeq(counts, x, sizeFactors=sizeFactors, engine=engine, useOptim=False, betaPrior=True,
                          factors=factors)
    dv = DP.DESeq_device(D.to_gene_major(counts, torch.device(dev)), x, sizeFactors, useOptim=False, betaPrior=True,
                         factors=factors)
    idx = dv["idx"].cpu().numpy()
    assert np.array_equal(idx, np.flatnonzero(~host["allZero"]))
    assert np.array_equal(dv["modelMatrix"], host["modelMatrix"])
    assert np.max(rel_err(dv["betaPriorVar"], host["betaPriorVar"])) < tol
    same = ((dv["dispGeneIter"].cpu().numpy() == host["dispGeneIter"][idx])
            & (dv["dispIter"].cpu().numpy() == host["dispIter"][idx]))
    if np.any(~same):
        # the dispersion steps are those of betaPrior=FALSE: the same knife-edge rule (decision margin below 4096
        # rounding bounds in the oracle) as test_device_pipeline_matches_host_pipeline
        from test_device_pipeline_gpu import _MarginOracle
        assert np.mean(~same) <= 0.01
        mo = _MarginOracle(oracle)
        pipeline.DESeq(counts, x, sizeFactors=sizeFactors, engine=mo, useOptim=False)
        margin = np.minimum(mo.margins[-2], mo.margins[-1])
        assert np.all(margin[~same] < 4096), (np.flatnonzero(~same)[:8], margin[~same][:8])
    e = rel_err(dv["dispersion"].cpu().numpy()[same], host["dispersion"][idx][same])
    assert np.max(e) < tol
    e = rel_err(dv["mleBetaMatrix"].cpu().numpy()[same], host["mleBetaMatrix"][idx][same], floor=1e-6)
    assert np.max(e) < tol, np.max(e)
    conv = (host["betaConv"][idx] == 1) & same
    it_same = dv["betaIter"].cpu().numpy()[conv] == host["betaIter"][idx][conv]
    assert np.mean(it_same) > 0.995
    for k in ("betaMatrix", "betaSE", "WaldStatistic", "deviance"):
        floor = 1e-6 if k != "deviance" else 1e-12
        e = rel_err(dv[k].cpu().numpy()[conv], host[k][idx][conv], floor=floor)
        assert np.max(e) < tol, (k, np.max(e))
    e = np.abs(dv["WaldPvalue"].cpu().numpy()[conv] - host["WaldPvalue"][idx][conv])
    assert np.max(e) < tol
    assert dv["betaMatrix"].shape[1] == x.shape[1] + len(factors)
    return host, dv


@pytest.mark.parametrize("name,factors", [("factor4", [_factor(40, 4)]),
                                          ("two_factors", [np.arange(40) % 4, (np.arange(40) // 4) % 2])])
def test_device_pipeline_beta_prior_matches_host(emu_dev, oracle, name, factors):
    from deseq2_b200 import pipeline, synth
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(300, 40, x=x, seed=23)
    _compare_pipelines(emu_dev, oracle, d["counts"], x, factors, d["sizeFactors"], "cpu")


def test_beta_prior_argument_errors(emu_dev):
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    factors = [_factor(12, 3)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(50, 12, x=x, seed=2)
    y = D.to_gene_major(d["counts"], torch.device("cpu"))
    for fn, arg in ((DP.DESeq_device, y), (pipeline.DESeq, d["counts"])):
        with pytest.raises(ValueError):
            fn(arg, x, d["sizeFactors"], betaPrior=True)
        with pytest.raises(ValueError):
            fn(arg, synth.design_factor(12, 4), d["sizeFactors"], betaPrior=True, factors=factors)
        with pytest.raises(ValueError):
            fn(arg, x, d["sizeFactors"], betaPrior=True, factors=factors, minReplicatesForReplace=7)


def _sharded_data(n, m, levels):
    from deseq2_b200 import pipeline, synth
    factors = [_factor(m, levels)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(n, m, x=x, seed=91)
    return d["counts"], x, d["sizeFactors"], factors


def _sharded_rank(rank, world, dev, n, m, levels):
    from deseq2_b200 import sharded
    K, x, sf, factors = _sharded_data(n, m, levels)
    lo, hi = sharded.shard_bounds(n, world, rank)
    y = gm(K[lo:hi], dev)
    plain = sharded.sharded_DESeq_device(y, x, sf)
    r = sharded.sharded_DESeq_device(y, x, sf, betaPrior=True, factors=factors)
    return {"betaPriorVar": r["betaPriorVar"], "gathered": r["gathered"],
            "extra_collectives": r["collectives"] - plain["collectives"], "n_local": r["idx"].numel()}


def _check_sharded(backend, n, m, levels, world=2):
    """The prior variance is estimated from every gene's MLE coefficients (one extra packed all-gather), so
    betaPriorVar and every gathered MAP result equal the single-process run bit for bit."""
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_sharded_rank, n, m, levels, world=world, backend=backend)
    K, x, sf, factors = _sharded_data(n, m, levels)
    whole = DP.DESeq_device(gm(K, DEVICE[backend]), x, sf, betaPrior=True, factors=factors)
    for g in got:
        assert 0 < g["n_local"] < whole["idx"].numel()
        assert g["extra_collectives"] == 1
        assert np.array_equal(g["betaPriorVar"], whole["betaPriorVar"])
        for k in ("betaMatrix", "betaSE", "WaldPvalue"):
            assert np.array_equal(g["gathered"][k], whole[k].cpu().numpy(), equal_nan=True), k


def test_sharded_beta_prior_equals_whole(emu_dev):
    _check_sharded("gloo", 400, 12, 3)


# ---------------------------------------------------------------- GPU (or the emulator with B200NB_LIB)

@pytest.mark.gpu
@pytest.mark.parametrize("design,n,m", [("factor10", 1500, 120), ("batch", 3000, 36), ("factor10", 600, 420)])
def test_device_pipeline_beta_prior_matches_host_gpu(engine, oracle, design, n, m):
    from deseq2_b200 import pipeline, synth
    factors = [_factor(m, 10)] if design == "factor10" else _bc_factors(m)
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(n, m, x=x, seed=11)
    _compare_pipelines(engine, oracle, d["counts"], x, factors, d["sizeFactors"], DEV)


@pytest.mark.gpu
def test_get_contrast_on_expanded_map_results(engine):
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    factors = [_factor(40, 4)]
    x = pipeline.factorDesign(factors)[0]
    d = synth.make_example_counts(800, 40, x=x, seed=31)
    dev = torch.device(DEV)
    y = D.to_gene_major(d["counts"], dev)
    dv = DP.DESeq_device(y, x, d["sizeFactors"], useOptim=False, betaPrior=True, factors=factors)
    idx = dv["idx"].cpu().numpy()
    ynz = y[dv["idx"]].contiguous()
    xe, pv = dv["modelMatrix"], dv["betaPriorVar"]
    counts = d["counts"][idx]
    nf = np.broadcast_to(d["sizeFactors"][None, :], counts.shape)
    disp = dv["dispersion"].cpu().numpy()
    beta = dv["betaMatrix"].cpu().numpy()
    for i, j in ((2, 1), (4, 2), (3, 1)):              # level i - 1 vs level j - 1 of the expanded columns
        con = np.zeros(xe.shape[1])
        con[i], con[j] = 1.0, -1.0
        g = DP.getContrast_device(ynz, xe, d["sizeFactors"], dv["dispersion"], dv["betaMatrix"], con, betaPriorVar=pv)
        h = pipeline.getContrast(counts, nf, xe, disp, beta, con, betaPriorVar=pv, engine=engine)
        for k in ("log2FoldChange", "lfcSE", "stat"):
            assert np.max(rel_err(g[k].cpu().numpy(), h[k], floor=1e-6)) < 1e-6, k
        assert np.max(np.abs(g["pvalue"].cpu().numpy() - h["pvalue"])) < 1e-6


@pytest.mark.gpu
def test_config4_size(engine):
    """BASELINE config 4: 50 000 genes x 1000 samples, a 10-level factor, betaPrior=TRUE."""
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    n, m = (50000, 1000) if DEV == "cuda" else (2000, 100)
    factors = [_factor(m, 10)]
    x = pipeline.factorDesign(factors)[0]
    assert np.array_equal(x, synth.design_factor(m, 10))
    d = synth.make_example_counts(n, m, x=x, seed=4)
    dv = DP.DESeq_device(D.to_gene_major(d["counts"], torch.device(DEV)), x, d["sizeFactors"], betaPrior=True,
                         factors=factors)
    pv = dv["betaPriorVar"]
    assert np.all(np.isfinite(pv)) and np.all(pv > 0)
    bm = dv["baseMean"].cpu().numpy()
    dispFit = dv["dispFit"].cpu().numpy()
    ref = _host_expanded(dv["mleBetaMatrix"].cpu().numpy(), factors, bm, dispFit)
    assert np.max(rel_err(pv, ref, floor=1e-300)) <= 1e-12
    for k in ("betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue", "deviance", "mleBetaMatrix"):
        assert torch.isfinite(dv[k]).all(), k
    assert (dv["betaIter"] < 100).double().mean().item() >= 0.99


@pytest.mark.gpu
def test_sharded_beta_prior_over_nccl_equals_whole(engine):
    _check_sharded("nccl", 20000, 60, 6, nccl_world())
