"""DESeq() with gene-specific normalization factors on the device: normalization_factors (b200nb_size_factors_norm_dev)
against pipeline.estimateNormFactors, the nf prep and Cook's kernels (b200nb_prep_nf_dev, b200nb_cooks_nf_dev) against
the host restatement, DESeq_device / nbinomLRT_device / getContrast_device with normalizationFactors against
pipeline.DESeq / nbinomLRT / getContrast driving the oracle engine, the constant-row property (an nf matrix whose
every row is s gives the sizeFactors=s results), a tximport-like property and the gene-sharded run.
The CPU tests run the engine's CUDA source on the SIMT emulator (`emu` fixture); the `-m gpu` tests run on a GPU, or on
the emulator when B200NB_LIB points at it."""
import warnings

import numpy as np
import pytest
import torch

from helpers import DEV, emu_dev, gm, gm64, rel_err
from ranks import DEVICE, nccl_world, run_ranks


def _make(n, x, seed):
    from deseq2_b200 import synth
    return synth.make_example_counts(n, x.shape[0], x=x, seed=seed, betaSD=0.3)


def _tx_nf(counts, sf, seed, sd=0.3):
    """tximport-like factors: the size factors times a per-entry length effect, row geometric mean of the effect 1."""
    rng = np.random.default_rng(seed)
    eff = np.exp(rng.normal(0.0, sd, counts.shape))
    eff /= np.exp(np.log(eff).mean(axis=1))[:, None]
    return sf[None, :] * eff


def _design(name):
    from deseq2_b200 import synth
    return {"condition12": lambda: synth.design_condition(12),
            "batch_condition36": lambda: synth.design_batch_condition(36, 3),
            "factor6_40": lambda: synth.design_factor(40, 6),
            "factor10_300": lambda: synth.design_factor(300, 10),
            "continuous40": lambda: np.c_[np.ones(40), np.linspace(-1.0, 1.0, 40)]}[name]()


# ---------------------------------------------------------------- factor estimation

@pytest.mark.parametrize("source", ["normMatrix", "avgTxLength"])
@pytest.mark.parametrize("type_", ["ratio", "poscounts"])
def test_normalization_factors_match_host(emu_dev, source, type_):
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = synth.design_condition(10)
    d = _make(300, x, 3)
    counts = d["counts"].astype(np.float64)
    counts[np.random.default_rng(1).random(counts.shape) < 0.05] = 0.0      # zeros: "ratio" drops those genes
    counts[4] = 0.0
    mat = np.exp(np.random.default_rng(2).normal(0.5, 0.4, counts.shape))
    y = gm64(counts, "cpu")
    got = DP.normalization_factors(y, 10, type=type_, **{source: gm64(mat, "cpu")})
    nm = mat if source == "normMatrix" else mat / np.exp(np.log(mat).mean(axis=1))[:, None]
    want = pipeline.estimateNormFactors(counts, nm, type=type_)
    nf = got["normalizationFactors"].numpy()
    assert np.max(rel_err(nf[:, :10], want)) < 1e-13
    assert np.all(nf[:, 10:] == 1.0)


def test_normalization_factors_reference_case(emu_dev):
    """The reference's test_size_factor.R: counts = 2 m * true.sf with nm = m / rowGeoMean(m) gives nf / nm = true.sf
    on the first row."""
    from deseq2_b200 import device_pipeline as DP
    m = np.arange(1, 17, dtype=np.float64).reshape(4, 4, order="F")
    nm = m / np.exp(np.log(m).mean(axis=1))[:, None]
    true_sf = np.array([2.0, 1.0, 1.0, 0.5])
    counts = 2.0 * m * true_sf[None, :]
    got = DP.normalization_factors(gm64(counts, "cpu"), 4, normMatrix=gm64(nm, "cpu"))
    nf = got["normalizationFactors"].numpy()[:, :4]
    assert np.allclose((nf / nm)[0], true_sf, rtol=1e-14, atol=0)


def test_normalization_factors_errors(emu_dev):
    from deseq2_b200 import device_pipeline as DP
    counts = np.random.default_rng(0).integers(1, 50, (20, 6)).astype(np.float64)
    y = gm64(counts, "cpu")
    good = gm64(np.ones((20, 6)), "cpu")
    with pytest.raises(ValueError, match="exactly one"):
        DP.normalization_factors(y, 6)
    with pytest.raises(ValueError, match="exactly one"):
        DP.normalization_factors(y, 6, normMatrix=good, avgTxLength=good)
    for v in (0.0, -1.0, np.nan, np.inf):
        bad = good.clone()
        bad[3, 2] = v
        with pytest.raises(ValueError, match="finite and positive"):
            DP.normalization_factors(y, 6, normMatrix=bad)
        with pytest.raises(ValueError, match="finite and positive"):
            DP.normalization_factors(y, 6, avgTxLength=bad)
    zeros = counts.copy()
    zeros[:, 0] = 0.0
    with pytest.raises(ValueError, match="every gene contains at least one zero"):
        DP.normalization_factors(gm64(zeros, "cpu"), 6, normMatrix=good)


# ---------------------------------------------------------------- kernels

@pytest.mark.parametrize("design", ["condition12", "continuous40", "factor10_300"])
def test_prep_nf_matches_host(emu_dev, design):
    """Short rows take prep_kernel<NF>, the 10-level factor at m = 300 the grouped one (m p >= 1024)."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    x = _design(design)
    m = x.shape[0]
    d = _make(60, x, 5)
    counts = d["counts"].astype(np.float64)
    counts[[3, 17]] = 0.0                                              # all-zero rows
    nf = _tx_nf(counts, d["sizeFactors"], 7)
    nz = counts.sum(axis=1) > 0
    xim = float(np.mean(1.0 / nf[nz].mean(axis=0)))
    pr = DP.prep(gm64(counts, "cpu"), x, None, normalizationFactors=gm64(nf, "cpu"), xim=xim)
    mv = pipeline.getBaseMeansAndVariances(counts, nf)
    norm = counts / nf
    with np.errstate(divide="ignore", invalid="ignore"):
        a0 = np.fmin(np.fmax(1e-8, np.fmin(pipeline.roughDispEstimate(norm, x),
                                           pipeline.momentsDispEstimate(mv["baseMean"], mv["baseVar"], nf[nz]))),
                     max(10, m))
    Q, R = np.linalg.qr(x)
    beta0 = np.linalg.solve(R, Q.T @ np.log(norm + 0.1).T)
    assert np.max(rel_err(pr["baseMean"].numpy(), mv["baseMean"])) < 1e-12
    assert np.max(rel_err(pr["baseVar"].numpy(), mv["baseVar"])) < 1e-12
    assert np.max(rel_err(pr["alpha0"].numpy()[nz], a0[nz])) < 1e-12
    assert np.array_equal(pr["allZero"].numpy() != 0, ~nz)
    # the kernel applies (X'X)^-1 X' (as for size factors); R's QR solve agrees to rounding of the two algorithms
    assert np.max(rel_err(pr["beta0"].numpy(), DP._projection(x) @ np.log(norm + 0.1).T, floor=1e-3)) < 1e-12
    assert np.max(rel_err(pr["beta0"].numpy(), beta0, floor=1e-3)) < 1e-10
    if pipeline.modelMatrixGroups(x) == x.shape[1]:
        mu = np.maximum(pipeline.linearModelMu(norm, x) * nf, 0.5)
        assert np.max(rel_err(pr["mu_lin"].numpy()[:, :m], mu)) < 1e-12


@pytest.mark.parametrize("design", ["condition12", "condition600", "continuous20"])
def test_cooks_nf_matches_host(emu_dev, design):
    """Cells of <= 256 samples (compact trimmed means), a cell of 300 (> 256: extraction path), no cell of 3."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = {"condition12": lambda: synth.design_condition(12), "condition600": lambda: synth.design_condition(600),
         "continuous20": lambda: np.c_[np.ones(20), np.linspace(-1.0, 1.0, 20)]}[design]()
    m = x.shape[0]
    d = _make(40, x, 9)
    counts = d["counts"].astype(np.float64)
    nf = _tx_nf(counts, d["sizeFactors"], 3)
    rng = np.random.default_rng(4)
    mu = nf * (counts / nf).mean(axis=1)[:, None] * np.exp(rng.normal(0, 0.1, counts.shape)) + 0.5
    H = rng.uniform(0.01, 0.5, counts.shape)
    ck = DP.cooks(gm64(counts, "cpu"), gm64(mu, "cpu"), gm64(H, "cpu"), x, None, normalizationFactors=gm64(nf, "cpu"))
    want = pipeline.calculateCooksDistance(counts, mu, H, nf, x)
    assert np.max(rel_err(ck["cooks"].numpy()[:, :m], want)) < 1e-12
    assert np.max(rel_err(ck["robustDisp"].numpy(), pipeline.robustMethodOfMomentsDisp(counts, nf, x))) < 1e-12
    mc = pipeline.recordMaxCooks(x, want)
    assert np.array_equal(np.isnan(ck["maxCooks"].numpy()), np.isnan(mc))
    ok = ~np.isnan(mc)
    assert np.max(rel_err(ck["maxCooks"].numpy()[ok], mc[ok]), initial=0.0) < 1e-12


# ---------------------------------------------------------------- constant rows = size factors

_KEYS = ("baseMean", "dispGeneEst", "dispFit", "dispMAP", "dispersion", "betaMatrix", "betaSE", "WaldStatistic",
         "WaldPvalue", "deviance", "maxCooks")


def _close(a, b, tol=1e-10, floor=1e-8):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    assert np.array_equal(np.isnan(a), np.isnan(b))
    ok = ~np.isnan(a)
    return np.max(rel_err(a[ok], b[ok], floor=floor), initial=0.0) < tol


@pytest.mark.parametrize("variant", ["plain", "betaPrior", "replace"])
def test_constant_rows_equal_size_factors(emu_dev, variant):
    from deseq2_b200 import device_pipeline as DP, synth
    if variant == "betaPrior":
        factors = [np.repeat([0, 1, 2], 6), np.tile([0, 1], 9)]
        x = __import__("deseq2_b200.pipeline").pipeline.factorDesign(factors)[0]
        kw = dict(betaPrior=True, factors=factors)
    else:
        x = synth.design_condition(16)
        kw = dict(minReplicatesForReplace=7) if variant == "replace" else {}
    m = x.shape[0]
    d = _make(200, x, 12)
    counts = d["counts"].copy()
    counts[6] = 0
    if variant == "replace":
        counts[[10, 20, 30], [1, 2, 9]] = 40 * counts[[10, 20, 30]].max(axis=1) + 200
    sf = d["sizeFactors"]
    y = gm64(counts, "cpu")
    a = DP.DESeq_device(y, x, sf, **kw)
    b = DP.DESeq_device(y, x, normalizationFactors=gm64(np.broadcast_to(sf, counts.shape), "cpu"), **kw)
    assert torch.equal(a["idx"], b["idx"])
    if variant == "replace":
        assert a["n_replaced"] == b["n_replaced"] > 0
    for k in _KEYS:
        assert _close(a[k], b[k]), k
    assert b["sizeFactors"] is None and b["normalizationFactors"].shape == (len(b["idx"]), y.shape[1])


def test_constant_rows_equal_size_factors_lrt_contrast(emu_dev):
    from deseq2_b200 import device_pipeline as DP, synth
    x = synth.design_batch_condition(18, 3)
    d = _make(150, x, 14)
    counts = d["counts"][d["counts"].sum(axis=1) > 0]
    sf = d["sizeFactors"]
    y = gm64(counts, "cpu")
    nf = gm64(np.broadcast_to(sf, counts.shape), "cpu")
    disp = torch.as_tensor(np.random.default_rng(0).uniform(0.05, 0.5, len(counts)))
    for xr in (x[:, :3], np.ones((18, 1))):
        a = DP.nbinomLRT_device(y, x, xr, sf, disp)
        b = DP.nbinomLRT_device(y, x, xr, None, disp, normalizationFactors=nf)
        for k in ("LRTStatistic", "LRTPvalue", "deviance", "betaMatrix", "betaSE"):
            assert torch.equal(a[k], b[k]), k                          # no xim involved: the same bits
    r = DP.DESeq_device(y, x, sf)
    for con in ([0, 1, -1, 0], [0, 0, 0, 1]):
        a = DP.getContrast_device(y, x, sf, r["dispersion"], r["betaMatrix"], con)
        b = DP.getContrast_device(y, x, None, r["dispersion"], r["betaMatrix"], con, normalizationFactors=nf)
        for k in ("log2FoldChange", "lfcSE", "stat", "pvalue"):
            assert torch.equal(a[k], b[k]), k


# ---------------------------------------------------------------- device vs host pipeline

def _compare_nf(engine, counts, x, nf, dev, tol=1e-6, **kw):
    """The acceptance rule of test_device_pipeline_matches_host_pipeline: every gene whose two dispersion line searches
    took the same number of steps on both sides agrees within tol; the others must be rare and oracle-certified knife
    edges (decision margin below 4096 rounding bounds)."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    host = pipeline.DESeq(counts, x, engine=engine, useOptim=False, normalizationFactors=nf, **kw)
    dv = DP.DESeq_device(gm64(counts, dev), x, useOptim=False, normalizationFactors=gm64(nf, dev), **kw)
    idx = dv["idx"].cpu().numpy()
    assert np.array_equal(idx, host["idx"])
    assert np.max(rel_err(dv["baseMean"].cpu().numpy(), host["baseMean"][idx])) < 1e-12
    assert np.max(rel_err(dv["trendCoefs"].cpu().numpy(), host["trendCoefs"])) < tol
    same = ((dv["dispGeneIter"].cpu().numpy() == host["dispGeneIter"][idx])
            & (dv["dispIter"].cpu().numpy() == host["dispIter"][idx]))
    if np.any(~same):
        from test_device_pipeline_gpu import _MarginOracle
        assert np.mean(~same) <= 0.02
        mo = _MarginOracle(engine)
        pipeline.DESeq(counts, x, engine=mo, useOptim=False, normalizationFactors=nf, **kw)
        margin = np.minimum(mo.margins[-2], mo.margins[-1])
        assert np.all(margin[~same] < 4096), (np.flatnonzero(~same)[:8], margin[~same][:8])
    for k in ("dispGeneEst", "dispMAP", "dispersion"):
        assert np.max(rel_err(dv[k].cpu().numpy()[same], host[k][idx][same])) < tol, k
    conv = (host["betaConv"][idx] == 1) & same
    for k in ("betaMatrix", "betaSE", "WaldStatistic", "deviance"):
        e = rel_err(dv[k].cpu().numpy()[conv], host[k][idx][conv], floor=1e-6 if k != "deviance" else 1e-12)
        assert np.max(e) < tol, (k, np.max(e))
    assert np.max(np.abs(dv["WaldPvalue"].cpu().numpy()[conv] - host["WaldPvalue"][idx][conv])) < tol
    mc_d, mc_h = dv["maxCooks"].cpu().numpy()[same], host["maxCooks"][idx][same]
    ok = ~np.isnan(mc_h)
    assert np.array_equal(np.isnan(mc_d), ~ok)
    assert np.max(rel_err(mc_d[ok], mc_h[ok]), initial=0.0) < tol
    return host, dv


@pytest.mark.parametrize("design", ["condition12", "batch_condition36", "factor6_40", "continuous40"])
def test_device_pipeline_nf_matches_host(emu_dev, oracle, design):
    x = _design(design)
    d = _make(240, x, 13)
    counts = d["counts"].copy()
    counts[5] = 0
    _compare_nf(oracle, counts, x, _tx_nf(counts, d["sizeFactors"], 8), "cpu")


def test_device_pipeline_nf_matches_host_beta_prior_and_replace(emu_dev, oracle):
    from deseq2_b200 import pipeline, synth
    factors = [np.repeat([0, 1, 2], 6), np.tile([0, 1], 9)]
    x = pipeline.factorDesign(factors)[0]
    d = _make(240, x, 15)
    _compare_nf(oracle, d["counts"], x, _tx_nf(d["counts"], d["sizeFactors"], 9), "cpu", betaPrior=True,
                factors=factors)
    x = synth.design_condition(16)
    d = _make(240, x, 16)
    counts = d["counts"].copy()
    counts[[10, 20, 30, 40], [1, 2, 9, 12]] = 40 * counts[[10, 20, 30, 40]].max(axis=1) + 200
    host, dv = _compare_nf(oracle, counts, x, _tx_nf(counts, d["sizeFactors"], 10), "cpu", minReplicatesForReplace=7)
    assert dv["n_replaced"] == host["n_replaced"] > 0


def test_lrt_and_contrast_nf_match_host(emu_dev, oracle):
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = synth.design_batch_condition(36, 3)
    d = _make(200, x, 31)
    counts = d["counts"][d["counts"].sum(axis=1) > 0]
    nf = _tx_nf(counts, d["sizeFactors"], 11)
    y, nfd = gm64(counts, "cpu"), gm64(nf, "cpu")
    disp = np.random.default_rng(3).uniform(0.05, 0.5, len(counts))
    g = DP.nbinomLRT_device(y, x, x[:, :3], None, torch.as_tensor(disp), normalizationFactors=nfd, useOptim=False)
    h = pipeline.nbinomLRT(counts, nf, x, x[:, :3], disp, engine=oracle, useOptim=False)
    conv = h["fullBetaConv"] & h["reducedBetaConv"]
    for k in ("LRTStatistic", "deviance", "betaMatrix"):
        e = rel_err(g[k].cpu().numpy()[conv], h[k][conv], floor=1e-6)
        assert np.max(e) < 1e-6, (k, np.max(e))
    beta = g["betaMatrix"]
    for con in ([0, 1, -1, 0], [0, 0, 0, 1], [0, 0.5, 0.5, -1]):
        a = DP.getContrast_device(y, x, None, torch.as_tensor(disp), beta, con, normalizationFactors=nfd)
        b = pipeline.getContrast(counts, nf, x, disp, beta.numpy(), con, engine=oracle)
        for k in ("log2FoldChange", "lfcSE", "stat"):
            assert np.max(rel_err(a[k].numpy(), b[k], floor=1e-6)) < 1e-6, k


def test_tximport_like_length_change(emu_dev):
    """Genes whose only change between the conditions is their transcript length: with the avgTxLength factors the
    log2 fold change is ~0, with size factors alone it is the length ratio."""
    from deseq2_b200 import device_pipeline as DP, synth
    x = synth.design_condition(12)
    d = synth.make_example_counts(400, 12, x=x, seed=21, betaSD=0.0, interceptMean=8)
    length = np.ones((400, 12))
    length[:100, x[:, 1] == 1] = 2.0                                   # first 100 genes: twice as long in B
    rng = np.random.default_rng(5)
    lam = 2.0 ** rng.normal(8, 1, 400)[:, None] * d["sizeFactors"][None, :] * length
    size = 1.0 / rng.uniform(0.02, 0.2, 400)[:, None]                    # NB dispersions 0.02 .. 0.2
    counts = rng.negative_binomial(size, size / (size + lam)).astype(np.int64)
    y = gm64(counts, "cpu")
    tx = DP.DESeq_device(y, x, avgTxLength=gm64(length, "cpu"))
    sf = DP.DESeq_device(y, x)
    lfc_tx, lfc_sf = tx["betaMatrix"][:, 1].numpy(), sf["betaMatrix"][:, 1].numpy()
    assert abs(np.median(lfc_tx[:100])) < 0.05                        # centred on 0, like the unchanged genes
    assert abs(np.median(lfc_tx[100:])) < 0.05
    assert np.median(lfc_sf[:100]) > 0.6        # most of log2(2); the size factors absorb part of it
    assert np.mean(np.abs(lfc_tx[:100]) < np.abs(lfc_sf[:100])) > 0.9


def test_nf_errors(emu_dev):
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = synth.design_condition(12)
    d = _make(40, x, 2)
    y = gm64(d["counts"], "cpu")
    nf = gm64(np.ones(d["counts"].shape), "cpu")
    with pytest.raises(ValueError, match="normalizationFactors must be a contiguous"):
        DP.DESeq_device(y, x, normalizationFactors=nf[:10])
    with pytest.raises(ValueError, match="float64 tensor"):
        DP.DESeq_device(y, x, normalizationFactors=nf.to(torch.float32))
    for v in (0.0, -2.0, np.nan, np.inf):
        bad = nf.clone()
        bad[1, 3] = v
        with pytest.raises(ValueError, match="finite and positive"):
            DP.DESeq_device(y, x, normalizationFactors=bad)
    with pytest.raises(ValueError, match="not both"):
        DP.DESeq_device(y, x, d["sizeFactors"], normalizationFactors=nf)
    with pytest.raises(ValueError, match="weights together with normalization factors"):
        DP.DESeq_device(y, x, normalizationFactors=nf, weights=torch.ones_like(nf))
    with pytest.raises(ValueError, match="not both"):
        DP.DESeq_device(y, x, normalizationFactors=nf, avgTxLength=nf)
    with pytest.raises(ValueError, match="not both"):
        DP.nbinomLRT_device(y, x, x[:, :1], d["sizeFactors"], torch.full((40,), 0.1), normalizationFactors=nf)
    with pytest.raises(ValueError, match="finite and positive"):
        DP.getContrast_device(y, x, None, torch.full((40,), 0.1), torch.zeros(40, 2), [0, 1],
                              normalizationFactors=nf * 0)
    with pytest.raises(ValueError):
        pipeline.DESeq(d["counts"], x, sizeFactors=d["sizeFactors"], normalizationFactors=np.ones(d["counts"].shape))


# ---------------------------------------------------------------- sharding

def _sharded_data(n, m, seeds):
    from deseq2_b200 import synth
    x = synth.design_batch_condition(m, 3)
    d = synth.make_example_counts(n, m, x=x, seed=seeds[0])
    return d["counts"], x, d["sizeFactors"], _tx_nf(d["counts"], d["sizeFactors"], seeds[1])


def _sharded_rank(rank, world, dev, n, m, seeds):
    from deseq2_b200 import device_pipeline as DP, sharded
    K, x, sf, nf = _sharded_data(n, m, seeds)
    lo, hi = sharded.shard_bounds(n, world, rank)
    y, nfl = gm(K[lo:hi], dev), gm(nf[lo:hi], dev)
    warnings.simplefilter("ignore")
    plain = sharded.sharded_DESeq_device(y, x, sf)
    captured = {}
    real = DP.DESeq_device

    def spy(*a, **kw):
        captured["xim"] = kw.get("nfXim")
        return real(*a, **kw)

    DP.DESeq_device = spy
    r = sharded.sharded_DESeq_device(y, x, normalizationFactors=nfl)
    DP.DESeq_device = real
    errors = 0
    for kw in (dict(minReplicatesForReplace=7), dict(avgTxLength=nfl)):
        try:
            sharded.sharded_DESeq_device(y, x, normalizationFactors=None if "avgTxLength" in kw else nfl, **kw)
        except ValueError:
            errors += 1
    return {"gathered": r["gathered"], "extra_collectives": r["collectives"] - plain["collectives"],
            "xim": captured["xim"], "errors": errors, "n_local": r["idx"].numel()}


def _check_sharded(backend, n, m, seeds, world=2):
    """The nf matrix sharded by rows: the same xim bits on every rank, results within 1e-9 of the single-process run,
    one collective more than the size-factor run; nf with outlier replacement and avgTxLength raise.  seeds: of the
    counts and of the factors."""
    from deseq2_b200 import device_pipeline as DP
    got = run_ranks(_sharded_rank, n, m, seeds, world=world, backend=backend)
    K, x, _, nf = _sharded_data(n, m, seeds)
    dev = DEVICE[backend]
    whole = DP.DESeq_device(gm64(K, dev), x, normalizationFactors=gm64(nf, dev))
    xim = got[0]["xim"]
    nz = K.sum(axis=1) > 0
    assert xim is not None and abs(xim - np.mean(1.0 / nf[nz].mean(axis=0))) < 1e-14 * xim
    for g in got:
        assert g["xim"] == xim
        assert g["extra_collectives"] == 1
        assert g["errors"] == 2
        assert 0 < g["n_local"] < whole["idx"].numel()
        for k in ("dispersion", "betaMatrix", "betaSE", "WaldPvalue"):
            a, b = g["gathered"][k], whole[k].cpu().numpy()
            assert np.array_equal(np.isnan(a), np.isnan(b)), k
            assert np.max(rel_err(a, b, floor=1e-8), initial=0.0, where=~np.isnan(b)) < 1e-9, k


def test_sharded_nf_equal_whole(emu_dev):
    _check_sharded("gloo", 400, 12, (91, 4))


# ---------------------------------------------------------------- GPU (or the emulator with B200NB_LIB)

@pytest.mark.gpu
@pytest.mark.parametrize("design,n,m", [("condition", 2000, 100), ("factor10", 600, 420), ("condition", 2000, 1000)])
def test_device_pipeline_nf_matches_host_gpu(engine, oracle, design, n, m):
    from deseq2_b200 import synth
    x = synth.design_condition(m) if design == "condition" else synth.design_factor(m, 10)
    d = _make(n, x, 11)
    counts = d["counts"].copy()
    counts[7] = 0
    _compare_nf(oracle, counts, x, _tx_nf(counts, d["sizeFactors"], 12), DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C2", "C4"])
def test_config_sizes_with_nf(engine, config):
    """BASELINE C2 (50 000 x 100, ~condition) and C4 (50 000 x 1000, 10-level factor) with tximport-like factors."""
    from deseq2_b200 import device_pipeline as DP, synth
    m = 100 if config == "C2" else 1000
    n = 50000 if DEV == "cuda" else 1000
    x = synth.design_condition(m) if config == "C2" else synth.design_factor(m, 10)
    d = synth.make_example_counts(n, m, x=x, seed=4)
    dv = DP.DESeq_device(gm64(d["counts"], DEV), x, normalizationFactors=gm64(_tx_nf(d["counts"], d["sizeFactors"], 6),
                                                                            DEV))
    for k in ("dispersion", "betaMatrix", "betaSE", "WaldStatistic", "WaldPvalue", "deviance"):
        assert torch.isfinite(dv[k]).all(), k
    assert (dv["betaIter"] < 100).double().mean().item() >= 0.99


@pytest.mark.gpu
def test_sharded_nf_over_nccl_equals_whole(engine):
    # The ranks' xim (column sums added over the ranks, divided on the device) can differ from the single-process xim
    # in the last bit, and on some data that moves a few genes by more than 1e-9: with seeds (91, 4) at this size, two
    # dispersions by up to 3e-8 on an H100 80GB HBM3, even with one rank.  Seeds (5, 7) give the same xim bits there.
    _check_sharded("nccl", 20000, 60, (5, 7), nccl_world())
