"""Device-resident pipeline (SURVEY.md 8f rows 2-3): pre-step kernel, trend-fit kernel and the full on-device
DESeq() Wald path against the numpy restatement of the R callers (deseq2_b200/pipeline.py) driving the same engine."""
import numpy as np
import pytest

from helpers import DEV, beta_args, disp_args, make_case, rel_err

pytestmark = pytest.mark.gpu



def _setup(n, m, x=None, seed=1):
    import torch
    from deseq2_b200 import device as D, synth
    d = synth.make_example_counts(n, m, x=x, seed=seed)
    y = D.to_gene_major(d["counts"], torch.device(DEV))
    return d, y


@pytest.mark.parametrize("design", ["condition", "batch", "batch-long-rows", "factor10-long-rows", "covariates-long-rows"])
def test_prep_kernel_matches_numpy(engine, design, n=2000):
    """The `-long-rows` designs (m p >= 1024) take the per-group kernel when the design has <= 32 distinct rows
    (prep_grouped_kernel) and the streaming kernel otherwise (continuous covariates)."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    m = 30
    if design.endswith("long-rows"):
        m, n = 300, min(n, 300)
    if design == "condition":
        x = synth.design_condition(m)
    elif design.startswith("batch"):
        x = synth.design_batch_condition(m, 3)
    elif design.startswith("factor10"):
        x = synth.design_factor(m, 10)
    else:
        x = np.c_[synth.design_condition(m), np.random.default_rng(8).normal(0, 1, (m, 2))]
    d, y = _setup(n, m, x=x, seed=3)
    sf = d["sizeFactors"]
    pr = DP.prep(y, x, sf)
    counts = d["counts"]
    mv = pipeline.getBaseMeansAndVariances(counts, sf)
    nz = ~mv["allZero"]
    assert np.array_equal(pr["allZero"].cpu().numpy().astype(bool), mv["allZero"])
    assert np.max(rel_err(pr["baseMean"].cpu().numpy()[nz], mv["baseMean"][nz])) < 1e-12
    assert np.max(rel_err(pr["baseVar"].cpu().numpy()[nz], mv["baseVar"][nz])) < 1e-10
    norm = counts / sf
    rough = pipeline.roughDispEstimate(norm[nz], x)
    mom = pipeline.momentsDispEstimate(mv["baseMean"][nz], mv["baseVar"][nz], sf)
    a0 = np.minimum(np.maximum(1e-8, np.minimum(rough, mom)), max(10, m))
    assert np.max(rel_err(pr["alpha0"].cpu().numpy()[nz], a0, floor=1e-8)) < 1e-8
    mu = np.maximum(pipeline.linearModelMu(norm[nz], x) * sf, 0.5)
    assert np.max(rel_err(pr["mu_lin"].cpu().numpy()[nz][:, :m], mu)) < 1e-10
    Q, R = np.linalg.qr(x)
    b0 = np.linalg.solve(R, Q.T @ np.log(norm[nz] + 0.1).T).T
    assert np.max(np.abs(pr["beta0"].cpu().numpy().T[nz] - b0)) < 1e-10


def test_trend_kernel_matches_numpy(engine, n=20000):
    import torch
    from deseq2_b200 import device_pipeline as DP, pipeline
    rng = np.random.default_rng(0)
    means = 10 ** rng.uniform(0, 4, n)
    disps = (0.1 + 4 / means) * rng.gamma(8, 1 / 8, n)
    disps[rng.random(n) < 0.02] = 1e-8              # genes at the floor are excluded from the fit
    disps[rng.random(n) < 0.01] *= 40               # outliers trimmed by the residual rule
    ref = pipeline.parametricDispersionFit(means[disps > 1e-6], disps[disps > 1e-6])
    dev = torch.device(DEV)
    out = DP.trend_fit(torch.as_tensor(means, device=dev), torch.as_tensor(disps, device=dev)).cpu().numpy()
    assert out[2] == 0
    assert np.max(rel_err(out[:2], ref)) < 1e-8


class _MarginOracle:
    """The CPU oracle as a pipeline engine that also records, per fitDisp call, every gene's decision margin."""

    def __init__(self, oracle):
        self.o, self.margins = oracle, []
        self.fitDispGrid, self.fitBeta = oracle.fitDispGrid, oracle.fitBeta

    def fitDisp(self, **kw):
        r = self.o.fitDisp(**kw, with_margin=True)
        self.margins.append(r["margin"])
        return r


def test_long_rows_take_the_segmented_kernels_in_one_launch(engine, oracle):
    """From m = 400 samples on, the DEVICE entry points run designs with p <= 4 on the segmented general-p kernels
    (capi.cu::long_rows; the host entry points keep the small-p kernels): one launch instead of classify and the two
    design variants of the line search, switched off by B200NB_LONG_ROWS=0 (read per call), results equal to the
    small-p kernels' and the oracle's."""
    import os
    import torch
    from deseq2_b200 import _lib, device as D, synth
    m, n = 448, 160
    x = synth.design_batch_condition(m, 3)
    c = make_case(n, m, x=x, seed=77, betaSD=0.5)
    dev = torch.device(DEV)
    y = D.to_gene_major(c["counts"], dev)
    T = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=dev)
    alpha = np.clip(0.1 + 4 / c["baseMean"], 1e-8, m)
    o = oracle.fitBeta(**beta_args(c, alpha))
    mu = np.maximum(c["nf"] * np.exp(o["beta_mat"] @ x.T), 0.5)
    mud, la0 = D.to_gene_major(mu, dev), T(np.log(c["alpha0"]))
    L = _lib.lib()

    def disp():
        k0 = L.b200nb_kernel_launches()
        r = D.fit_disp(y, x, mud, la0, la0, 1.0, float(np.log(1e-9)), 1.0, 1e-6, 100, False)
        return {k: v.cpu().numpy() for k, v in r.items()}, L.b200nb_kernel_launches() - k0

    seg, n_seg = disp()
    os.environ["B200NB_LONG_ROWS"] = "0"
    try:
        small, n_small = disp()
    finally:
        os.environ.pop("B200NB_LONG_ROWS")
    assert (n_seg, n_small) == (1, 3)
    od = oracle.fitDisp(**disp_args(c, mu, np.log(c["alpha0"])), with_margin=True)
    same = (seg["iter"] == od["iter"]) & (seg["iter_accept"] == od["iter_accept"])
    assert np.all(same | (od["margin"] <= 64.0))
    assert np.max(rel_err(seg["log_alpha"][same], od["log_alpha"][same], floor=1e-3)) < 1e-6
    both = (seg["iter"] == small["iter"]) & (seg["iter_accept"] == small["iter_accept"])
    assert both.mean() > 0.97
    assert np.max(rel_err(seg["log_alpha"][both], small["log_alpha"][both], floor=1e-3)) < 1e-6
    lam = T(np.full(4, 1e-6) / np.log(2) ** 2)
    con = T(np.r_[1.0, 0, 0, 0])
    b = D.fit_beta(y, x, T(c["sf"]), T(alpha), con, T(c["beta0"].T), lam, 1e-8, 100)
    assert np.array_equal(b["iter"].cpu().numpy(), o["iter"])
    assert np.max(np.abs(b["beta_mat"].cpu().numpy().T - o["beta_mat"])) < 1e-6
    assert np.max(rel_err(b["hat_diagonals"].cpu().numpy()[:, :m], o["hat_diagonals"])) < 1e-6


@pytest.mark.parametrize("design,n,m", [("condition", 6000, 40), ("condition", 4000, 6), ("condition", 3000, 12),
                                        ("batch", 3000, 36), ("factor10", 1500, 120), ("batch", 600, 420)])
def test_device_pipeline_matches_host_pipeline(engine, oracle, design, n, m):
    """The device-resident DESeq() against the numpy restatement of the R glue driving the same engine through the C ABI:
    EVERY gene within 1e-6 on dispGeneEst / dispMAP / dispersion / beta / SE, unless its line search took a different
    number of steps -- which is only accepted for genes the oracle marks as knife-edge (decision margin below 4096
    rounding bounds: the two sides' pre-steps differ by rounding, numpy vs prep_kernel), and must be rare."""
    from deseq2_b200 import device_pipeline as DP, pipeline, synth
    x = {"condition": synth.design_condition(m), "batch": synth.design_batch_condition(m, 3),
         "factor10": synth.design_factor(m, 10)}[design]
    d, y = _setup(n, m, x=x, seed=11)
    host = pipeline.DESeq(d["counts"], x, sizeFactors=d["sizeFactors"], engine=engine, useOptim=False)
    dv = DP.DESeq_device(y, x, d["sizeFactors"], useOptim=False)
    idx = dv["idx"].cpu().numpy()
    assert np.array_equal(idx, np.flatnonzero(~host["allZero"]))
    assert np.max(rel_err(dv["trendCoefs"].cpu().numpy(), host["trendCoefs"])) < 1e-6
    assert abs(dv["dispPriorVar"] - host["dispPriorVar"]) < 1e-6 * max(1.0, host["dispPriorVar"])
    same = ((dv["dispGeneIter"].cpu().numpy() == host["dispGeneIter"][idx])
            & (dv["dispIter"].cpu().numpy() == host["dispIter"][idx]))
    print(f"\n{design} {n}x{m}: line-search step counts differ on {np.sum(~same)} of {len(same)} genes")
    for k in ("dispGeneEst", "dispMAP", "dispersion"):
        e = rel_err(dv[k].cpu().numpy(), host[k][idx])
        assert np.max(e[same]) < 1e-6, (k, np.max(e[same]), int(np.sum(e[same] >= 1e-6)))
    conv = (host["betaConv"][idx] == 1) & same
    assert np.array_equal(dv["betaIter"].cpu().numpy()[same], host["betaIter"][idx][same])
    e = rel_err(dv["betaMatrix"].cpu().numpy()[conv], host["betaMatrix"][idx][conv], floor=1e-6)
    assert np.max(e) < 1e-6, np.max(e)
    se = rel_err(dv["betaSE"].cpu().numpy()[conv], host["betaSE"][idx][conv])
    assert np.max(se) < 1e-6, np.max(se)
    # the p-values inherit the statistic's agreement: d log(2 Phi(-|z|)) / dz ~ -|z|, so a relative difference d in z
    # becomes about z^2 d in p.  The statistic is beta / SE, each within 1e-6 above: z agrees to 2e-6 relative.
    z, hz = dv["WaldStatistic"].cpu().numpy()[conv], host["WaldStatistic"][idx][conv]
    assert np.max(rel_err(z, hz, floor=1e-6)) < 2e-6
    pv, hp = dv["WaldPvalue"].cpu().numpy()[conv], host["WaldPvalue"][idx][conv]
    e = rel_err(pv, hp, floor=1e-300) / (2e-6 * (1.0 + hz ** 2))
    assert np.max(e) < 1, (np.max(e), hz[np.argmax(e)], pv[np.argmax(e)], hp[np.argmax(e)])
    if np.any(~same):
        assert np.mean(~same) < 0.005
        mo = _MarginOracle(oracle)
        pipeline.DESeq(d["counts"], x, sizeFactors=d["sizeFactors"], engine=mo, useOptim=False)
        margin = np.minimum(mo.margins[-2], mo.margins[-1])          # the MLE and the MAP line search of the same genes
        assert np.all(margin[~same] < 4096), (np.flatnonzero(~same)[:8], margin[~same][:8])
        e = rel_err(dv["dispersion"].cpu().numpy(), host["dispersion"][idx])
        assert np.max(e[~same]) < 5e-2


@pytest.mark.parametrize("design,m", [("condition", 12), ("condition", 60), ("batch", 36), ("covariate", 20),
                                      ("factor10", 200), ("condition", 150), ("condition", 400), ("condition", 700),
                                      ("covariate", 100), ("covariate", 300), ("factor10", 1000)])
def test_cooks_kernel_matches_numpy(engine, design, m, n=800):
    """SURVEY.md 8f row 1: robust moments dispersion (per-cell trimmed means), Cook's distances and their maximum
    (R/core.R:2277-2359) on device vs the numpy restatement."""
    import torch
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    rng = np.random.default_rng(5)
    if design == "condition":
        x = synth.design_condition(m)
    elif design == "batch":
        x = synth.design_batch_condition(m, 3)
    elif design == "factor10":
        x = synth.design_factor(m, 10)
    else:
        x = np.c_[np.ones(m), rng.normal(0, 1, m)]          # every sample its own cell -> trimmedVariance branch
    if m > 100:
        n = min(n, 200)     # cells of 33..256 samples (rank-counting trimmed means, 2 / 4 / 8 entries per lane) and beyond
    d = synth.make_example_counts(n, m, x=x if design != "covariate" else None, seed=17)
    counts = d["counts"][d["counts"].sum(axis=1) > 0]
    counts[::7, 0] *= 30                                    # planted outliers (test_outlier.R:33-55 idea)
    sf = d["sizeFactors"]
    n = len(counts)
    mu = np.maximum((counts / sf).mean(axis=1, keepdims=True) * sf[None, :] * rng.uniform(0.8, 1.25, (n, m)), 0.5)
    H = rng.uniform(0.01, 0.6, (n, m))
    dev = torch.device(DEV)
    out = DP.cooks(D.to_gene_major(counts, dev), D.to_gene_major(mu, dev), D.to_gene_major(H, dev), x, sf)
    ref_disp = pipeline.robustMethodOfMomentsDisp(counts, sf, x)
    ref_cooks = pipeline.calculateCooksDistance(counts, mu, H, sf, x)
    ref_max = pipeline.recordMaxCooks(x, ref_cooks)
    assert np.max(rel_err(out["robustDisp"].cpu().numpy(), ref_disp)) < 1e-10
    assert np.max(rel_err(out["cooks"].cpu().numpy()[:, :m], ref_cooks, floor=1e-12)) < 1e-9
    got_max = out["maxCooks"].cpu().numpy()
    if np.all(np.isnan(ref_max)):
        assert np.all(np.isnan(got_max))
    else:
        assert np.max(rel_err(got_max, ref_max, floor=1e-12)) < 1e-9


def test_lrt_device_matches_host(engine, n=3000):
    """BASELINE.json config 5's call sequence (nbinomLRT ~batch+condition vs ~batch) on device vs the host glue."""
    import torch
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    m = 40
    full = synth.design_batch_condition(m, 2)
    reduced = full[:, :2]
    d = synth.make_example_counts(n, m, x=full, seed=41, betaSD=0.7)
    counts = d["counts"][d["counts"].sum(axis=1) > 0]
    sf = d["sizeFactors"]
    nf = np.broadcast_to(sf[None, :], counts.shape)
    alpha = np.clip(0.1 + 4 / (counts / sf).mean(axis=1), 1e-8, m)
    host = pipeline.nbinomLRT(counts, nf, full, reduced, alpha, engine=engine)
    dev = torch.device(DEV)
    got = DP.nbinomLRT_device(D.to_gene_major(counts, dev), full, reduced, sf, torch.as_tensor(alpha, device=dev))
    ok = host["fullBetaConv"] & host["reducedBetaConv"]
    # the statistic is built from log-likelihoods at the UNCLAMPED means (R/fitNbinomGLMs.R:180-182): genes with fitted
    # means below minmu (zeros in a whole design cell) are part of the comparison
    assert ((counts / sf).min(axis=1) <= 0.5)[ok].sum() > 50
    st = got["LRTStatistic"].cpu().numpy()
    assert np.max(np.abs(st[ok] - host["LRTStatistic"][ok]) / (1 + np.abs(host["deviance"][ok]))) < 1e-9
    from scipy.stats import chi2
    # every p-value, the smallest included: a difference ds in the statistic moves log p by the chi-square hazard
    # f(s) / Q(s) times ds
    pv, hp, hs = got["LRTPvalue"].cpu().numpy()[ok], host["LRTPvalue"][ok], host["LRTStatistic"][ok]
    hazard = np.exp(chi2.logpdf(hs, host["df"]) - chi2.logsf(hs, host["df"]))
    tol = 1e-9 + 2.0 * hazard * np.abs(st[ok] - hs)
    assert np.all(np.abs(pv - hp) <= tol * hp + np.finfo(float).tiny), np.max(np.abs(pv - hp) / (tol * hp))
    assert np.min(hp) < 1e-12
    assert np.max(rel_err(got["betaMatrix"].cpu().numpy()[ok], host["betaMatrix"][ok], floor=1e-6)) < 1e-6


def test_optim_fallback_device_vs_host(engine, n=240):
    """R/fitNbinomGLMs.R:203-227, 340-407 (test_optim.R:29-39): rows whose IRLS does not converge are refitted by the
    box-constrained maximiser -- on the device (b200nb_beta_optim_dev) vs the host glue (scipy L-BFGS-B = R's optim).
    Both maximise the same strictly concave objective, so they meet at its unique maximiser; L-BFGS-B stops at
    factr = 1e7 (about 1e-5 in beta), the device Newton iteration goes on to ~1e-10, hence the tolerances."""
    import torch
    from deseq2_b200 import device as D, device_pipeline as DP, pipeline, synth
    m = 10
    x = synth.design_condition(m)
    d = synth.make_example_counts(n, m, x=x, seed=91)
    counts = d["counts"][d["counts"].sum(axis=1) > 0].copy()
    bad = np.arange(0, len(counts), 12)
    counts[bad] = np.array([0, 0, 0, 0, 0, 1000, 1000, 0, 0, 0])            # the reference's own divergent row
    counts[bad[::2], 5] = 3000                                             # ... and variations of it
    sf = d["sizeFactors"]
    nf = np.broadcast_to(sf[None, :], counts.shape)
    alpha = np.clip(0.1 + 4 / (counts / sf).mean(axis=1), 1e-8, m)
    raw = pipeline.fitNbinomGLMs(counts, nf, x, alpha, engine=engine, useOptim=False)
    assert (~raw["betaConv"][bad]).all(), "the planted rows must defeat the IRLS"
    host = pipeline.fitNbinomGLMs(counts, nf, x, alpha, engine=engine)       # useOptim = TRUE, the reference default
    dev = torch.device(DEV)
    y = D.to_gene_major(counts, dev)
    pr = DP.prep(y, x, sf, want_mu=False)
    LN2 = np.log(2.0)
    lam = torch.full((2,), 1e-6 / LN2 ** 2, dtype=torch.float64, device=dev)
    contrast = torch.tensor([1.0, 0.0], dtype=torch.float64, device=dev)
    ad = torch.as_tensor(alpha, device=dev)
    fb = D.fit_beta(y, pr["xd"], pr["sfd"], ad, contrast, pr["beta0"], lam, 1e-8, 100, want_mu=False)
    ll = D.nb_loglik(y, pr["xd"], pr["sfd"], ad, fb["beta_mat"], want_mu=True)
    conv, nopt = DP._optim_fallback(y, pr["xd"], pr["sfd"], ad, fb, pr["beta0"], lam, contrast, 100, 0.5, ll)
    rows = np.flatnonzero(~raw["betaConv"])
    assert nopt == len(rows) and set(bad) <= set(rows)
    conv = conv.cpu().numpy()
    assert conv[rows].all() and np.array_equal(conv, host["betaConv"] | conv)
    got_beta = (fb["beta_mat"] / LN2).T.cpu().numpy()
    got_se = (torch.sqrt(torch.clamp(fb["beta_var_mat"], min=0)) / LN2).T.cpu().numpy()
    got_ll = ll["logLike"].cpu().numpy()
    # the device optimum is at least as good as L-BFGS-B's, and the two agree to L-BFGS-B's own stopping accuracy
    assert np.all(got_ll[rows] >= host["logLike"][rows] - 1e-7 * (1 + np.abs(host["logLike"][rows])))
    assert np.max(np.abs(got_ll[rows] - host["logLike"][rows]) / (1 + np.abs(host["logLike"][rows]))) < 1e-6
    # The planted rows have a design cell of zeros: the likelihood is flat in that cell's coefficient beyond
    # mu ~ 1e-4 and only the 1e-6 ridge fixes it, so L-BFGS-B stops (factr = 1e7) a unit or two short of the maximiser the
    # Newton iteration reaches.  What is identifiable must agree: the fitted means of the samples that carry counts.
    got_mu = ll["mu"].cpu().numpy()[:, :m]
    for r_ in rows:
        sel = host["mu"][r_] > 0.5
        assert sel.any()
        assert np.max(rel_err(got_mu[r_, sel], host["mu"][r_, sel])) < 1e-3, r_
        assert np.all(got_mu[r_, ~sel] < 1e-2)
        if np.max(np.abs(got_beta[r_] - host["betaMatrix"][r_])) < 1e-3:       # a fully identified row: SEs agree too
            assert np.max(rel_err(got_se[r_], host["betaSE"][r_])) < 5e-3
    assert np.all(np.abs(got_beta[rows]) <= 30.0 + 1e-9) and np.all(np.isfinite(got_se[rows]))
    # rows the IRLS did fit are untouched
    ok = raw["betaConv"]
    assert np.max(rel_err(got_beta[ok], raw["betaMatrix"][ok], floor=1e-9)) < 1e-6
