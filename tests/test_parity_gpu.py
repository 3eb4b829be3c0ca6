"""GPU parity tests: the CUDA engine (through the C ABI, host buffers, exactly what the R shim would pass)
against the CPU oracle on identical seeded inputs.  Tolerances: 1e-6 relative on every floating-point output
(north_star), exact on iteration counters for every gene whose line-search decisions are not knife-edge
(oracle `margin` > 1e-9: two correct fp64 evaluations cannot legitimately disagree there)."""
import numpy as np
import pytest

from helpers import DISP_KEYS, beta_args, disp_args, make_case, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-6


def test_device_special_functions(engine):
    import ctypes as C

    import mpmath as mp
    from deseq2_b200 import _lib
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.uniform(1e-4, 40, 4000), 10 ** rng.uniform(-6, 9, 4000), np.arange(1, 200) * 0.5])
    lg, dg, tg = (np.empty_like(x) for _ in range(3))
    P = lambda a: C.c_void_p(a.ctypes.data)
    _lib.check(_lib.lib().b200nb_test_special(P(x), len(x), P(lg), P(dg), P(tg)), "test_special")
    mp.mp.dps = 40
    idx = rng.choice(len(x), 600, replace=False)
    for i in idx:
        xi = mp.mpf(float(x[i]))
        rl, rd, rt = float(mp.loggamma(xi)), float(mp.digamma(xi)), float(mp.polygamma(1, xi))
        # absolute accuracy on the scale max(1,|f|): lgamma/digamma cross zero at x = 1, 2 / 1.4616
        assert abs(lg[i] - rl) <= 2e-14 * max(1.0, abs(rl)), (x[i], lg[i], rl)
        assert abs(dg[i] - rd) <= 2e-14 * max(1.0, abs(rd)), (x[i], dg[i], rd)
        assert abs(tg[i] - rt) <= 2e-14 * max(1.0, abs(rt)), (x[i], tg[i], rt)


ROBUST = 64.0   # decision margin, in units of the a-priori fp64 rounding bound (see oracle_fit_disp)


def _compare_disp(g, o, name, min_robust=0.9):
    robust = o["margin"] > ROBUST
    same = (g["iter"] == o["iter"]) & (g["iter_accept"] == o["iter_accept"])
    # every gene whose decisions are not knife-edge must follow the oracle's control flow exactly
    bad = np.flatnonzero(~same & robust)
    assert bad.size == 0, (f"{name}: {bad.size} robust genes differ in iter/iter_accept, e.g. gene {bad[:5]} "
                           f"gpu iter {g['iter'][bad[:5]]} oracle iter {o['iter'][bad[:5]]} "
                           f"margin {o['margin'][bad[:5]]}")
    assert robust.mean() >= min_robust, f"{name}: only {robust.mean():.3f} of genes have robust decisions"
    sel = robust & same
    for k in DISP_KEYS if sel.any() else ():
        if k in ("last_dlp", "last_change", "last_d2lp", "initial_dlp"):
            # derivatives / differences of nearly equal numbers: absolute error on the scale of the posterior
            err = np.abs(g[k][sel] - o[k][sel]) / (np.abs(o["last_lp"][sel]) * 1e-3 + np.abs(o[k][sel]) + 1e-12)
        else:
            err = rel_err(g[k][sel], o[k][sel])
        assert np.nanmax(err) < TOL, f"{name}: {k} max rel err {np.nanmax(err):.3e}"
    assert not sel.any() or np.max(rel_err(np.exp(g["log_alpha"][sel]), np.exp(o["log_alpha"][sel]))) < TOL
    # knife-edge genes (either side may take the other branch): both must still end at the same posterior value
    rest = ~sel
    if rest.any():
        d = np.abs(g["last_lp"][rest] - o["last_lp"][rest]) / (1.0 + np.abs(o["last_lp"][rest]))
        assert np.nanmax(d) < 1e-5, f"{name}: knife-edge genes end at different posterior values ({np.nanmax(d):.2e})"
    return robust.mean(), same.mean()


@pytest.mark.parametrize("n,m,seed", [(3000, 100, 11), (1500, 6, 12), (800, 37, 13)])
def test_fit_disp_mle_parity(engine, oracle, n, m, seed):
    c = make_case(n, m, seed=seed)
    a = disp_args(c, c["mu"], np.log(c["alpha0"]))
    g = engine.fitDisp(**a)
    o = oracle.fitDisp(**a, with_margin=True)
    _compare_disp(g, o, f"mle {n}x{m}", min_robust=0.9 if m >= 30 else 0.3)


def test_fit_disp_map_parity(engine, oracle, n=3000):
    c = make_case(n, 100, seed=21)
    a0 = disp_args(c, c["mu"], np.log(c["alpha0"]))
    mle = oracle.fitDisp(**a0)
    fit = 0.1 + 4.0 / c["baseMean"]
    a = disp_args(c, c["mu"], mle["log_alpha"], prior_mean=np.log(fit), sigmasq=0.6, usePrior=True)
    _compare_disp(engine.fitDisp(**a), oracle.fitDisp(**a, with_margin=True), "map")


def test_fit_disp_f64_counts_and_no_cr(engine, oracle):
    c = make_case(500, 20, seed=22)
    a = disp_args(c, c["mu"], np.log(c["alpha0"]), useCR=False, y=c["counts"].astype(np.float64))
    _compare_disp(engine.fitDisp(**a), oracle.fitDisp(**a, with_margin=True), "f64/noCR", min_robust=0.5)


def test_fit_disp_grid_parity(engine, oracle):
    c = make_case(400, 30, seed=23)
    grid = np.linspace(np.log(1e-8), np.log(30), 20)
    kw = dict(ySEXP=c["counts"], xSEXP=c["x"], mu_hatSEXP=c["mu"], disp_gridSEXP=grid,
              log_alpha_prior_meanSEXP=np.log(0.1 + 4 / c["baseMean"]), log_alpha_prior_sigmasqSEXP=0.5,
              usePriorSEXP=True, weightsSEXP=None, useWeightsSEXP=False, weightThresholdSEXP=1e-2, useCRSEXP=True)
    g = engine.fitDispGrid(**kw)["log_alpha"]
    o = oracle.fitDispGrid(**kw)["log_alpha"]
    # argmax on a grid: identical grid point unless two grid values tie to rounding
    assert np.mean(np.abs(g - o) < 1e-9) > 0.995
    assert np.max(np.abs(g - o)) < 2.0 * (grid[1] - grid[0]) / 9.5


def _compare_beta(g, o, name, tol=TOL):
    assert np.array_equal(g["iter"], o["iter"]), f"{name}: iter differs on {np.sum(g['iter'] != o['iter'])} genes"
    for k in ("beta_mat", "beta_var_mat", "hat_diagonals", "contrast_num", "contrast_denom", "deviance"):
        err = rel_err(g[k], o[k], floor=1e-8)
        assert np.nanmax(err) < tol, f"{name}: {k} max rel err {np.nanmax(err):.3e}"
    se = rel_err(np.sqrt(g["beta_var_mat"]), np.sqrt(o["beta_var_mat"]))
    assert np.nanmax(se) < tol


@pytest.mark.parametrize("n,m,seed,useQR", [(3000, 100, 31, True), (1500, 6, 32, True), (800, 37, 33, False)])
def test_fit_beta_parity(engine, oracle, n, m, seed, useQR):
    c = make_case(n, m, seed=seed)
    alpha = np.clip(0.1 + 4.0 / c["baseMean"], 1e-8, 10)
    a = beta_args(c, alpha, useQR=useQR)
    _compare_beta(engine.fitBeta(**a), oracle.fitBeta(**a), f"beta {n}x{m}")


def test_fit_beta_maxit0_contrast(engine, oracle):
    """results() re-entry (R/results.R:797-807): maxit=0, numeric contrast, only the covariance block runs."""
    c = make_case(600, 24, seed=34)
    alpha = np.clip(0.1 + 4.0 / c["baseMean"], 1e-8, 10)
    fit = oracle.fitBeta(**beta_args(c, alpha))
    a = beta_args(c, alpha, beta0=fit["beta_mat"], maxit=0, useQR=False, contrast=np.array([0.0, 1.0]))
    g, o = engine.fitBeta(**a), oracle.fitBeta(**a)
    assert np.all(g["iter"] == 0)
    _compare_beta(g, o, "maxit0")


# ---------------------------------------------------------------- evaluation modes, weights, designs

def test_fit_disp_big_and_mixed_counts(engine, oracle, n=1200):
    """High-count genes (BIG mode: every count >= 10), mixed genes (GEN mode: max >= 256 and min < 10) and
    low-count genes (TAB mode) in one call."""
    c = make_case(n, 48, seed=41, interceptMean=8.0, interceptSD=3.0)
    y = c["counts"]
    big = np.flatnonzero(y.max(axis=1) >= 256)[:n // 15]     # force GEN mode: a few tiny counts in high-count genes
    y[big, :3] = np.arange(3 * len(big)).reshape(len(big), 3) % 7
    assert (y.min(axis=1) >= 10).sum() > n // 12 and ((y.max(axis=1) >= 256) & (y.min(axis=1) < 10)).sum() > n // 60
    assert (y.max(axis=1) < 256).sum() > n // 24
    a = disp_args(c, c["mu"], np.log(c["alpha0"]))
    _compare_disp(engine.fitDisp(**a), oracle.fitDisp(**a, with_margin=True), "modes", min_robust=0.85)


def test_fit_disp_non_integer_counts(engine, oracle):
    c = make_case(300, 16, seed=42)
    y = c["counts"].astype(np.float64) + 0.25
    a = disp_args(c, c["mu"], np.log(c["alpha0"]), y=y)
    _compare_disp(engine.fitDisp(**a), oracle.fitDisp(**a, with_margin=True), "non-integer y", min_robust=0.8)


def _weights_for(c, seed, p_small=0.08):
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.3, 1.0, c["counts"].shape)
    w[rng.random(w.shape) < p_small] = 1e-3          # below the Cox-Reid weightThreshold (1e-2)
    return np.maximum(w / w.max(axis=1, keepdims=True), 1e-6)


@pytest.mark.parametrize("design,seed", [("condition", 51), ("batch", 52), ("factor4", 53)])
def test_fit_disp_weights_and_designs(engine, oracle, design, seed):
    from deseq2_b200 import synth
    m = 24
    x = {"condition": synth.design_condition(m), "batch": synth.design_batch_condition(m, 2),
         "factor4": synth.design_factor(m, 4)}[design]
    c = make_case(500, m, x=x, seed=seed)
    alpha = np.clip(0.1 + 4 / c["baseMean"], 1e-8, m)
    mu = c["mu"] if c["mu"] is not None else np.maximum(
        c["nf"] * np.exp(oracle.fitBeta(**beta_args(c, alpha))["beta_mat"] @ x.T), 0.5)
    w = _weights_for(c, seed)
    a = disp_args(c, mu, np.log(c["alpha0"]), prior_mean=np.log(alpha), sigmasq=0.8, usePrior=True, weights=w,
                  useWeights=True)
    _compare_disp(engine.fitDisp(**a), oracle.fitDisp(**a, with_margin=True), f"weights/{design}", min_robust=0.85)


def test_fit_disp_weights_drop_a_design_column(engine, oracle):
    """Cox-Reid column removal (src/DESeq2.cpp:41-43): every sample of the second group below the weight
    threshold -> that design column is all zero on the kept rows and is dropped."""
    from deseq2_b200 import synth
    m = 12
    c = make_case(200, m, x=synth.design_condition(m), seed=54)
    w = np.ones(c["counts"].shape)
    w[:, m // 2:] = 5e-3
    a = disp_args(c, c["mu"], np.log(c["alpha0"]), weights=w, useWeights=True)
    _compare_disp(engine.fitDisp(**a), oracle.fitDisp(**a, with_margin=True), "dropped column", min_robust=0.8)


@pytest.mark.parametrize("design,seed,useQR", [("batch", 61, True), ("factor4", 62, False), ("intercept", 63, True)])
def test_fit_beta_designs_weights_nf_matrix(engine, oracle, design, seed, useQR):
    from deseq2_b200 import synth
    m = 24
    x = {"batch": synth.design_batch_condition(m, 2), "factor4": synth.design_factor(m, 4),
         "intercept": np.ones((m, 1))}[design]
    c = make_case(600, m, x=x if design != "intercept" else None, seed=seed)
    if design == "intercept":
        c["x"] = x
        c["beta0"] = np.log(c["baseMean"])[:, None]
    rng = np.random.default_rng(seed)
    nf = c["nf"] * np.exp(rng.normal(0, 0.2, c["nf"].shape))          # gene-specific normalisation factors
    nf /= np.exp(np.mean(np.log(nf), axis=1, keepdims=True))
    alpha = np.clip(0.1 + 4 / c["baseMean"], 1e-8, m)
    w = _weights_for(c, seed, p_small=0.0)
    p = x.shape[1]
    lam = np.full(p, 1e-6) / np.log(2) ** 2
    if p > 1:
        lam[-1] = 0.3
    a = beta_args(c, alpha, nf=nf, weights=w, useWeights=True, useQR=useQR, lam=lam, x=x,
                  contrast=np.r_[np.zeros(p - 1), 1.0])
    _compare_beta(engine.fitBeta(**a), oracle.fitBeta(**a), f"beta/{design}")


def test_fit_beta_badly_scaled_covariate(engine, oracle):
    """test_optim.R:2-26: a continuous covariate with sd 1000 -- the equilibrated Cholesky must track the QR branch."""
    rng = np.random.default_rng(71)
    m = 20
    x = np.c_[np.ones(m), rng.normal(0, 1000, m)]
    c = make_case(300, m, seed=72)
    c["x"] = x
    Q, R = np.linalg.qr(x)
    c["beta0"] = np.linalg.solve(R, Q.T @ np.log(c["counts"] / c["nf"] + 0.1).T).T
    alpha = np.clip(0.1 + 4 / c["baseMean"], 1e-8, m)
    a = beta_args(c, alpha, x=x)
    g, o = engine.fitBeta(**a), oracle.fitBeta(**a)
    conv = o["iter"] < 100
    assert np.array_equal(g["iter"][conv], o["iter"][conv])
    assert np.nanmax(rel_err(g["beta_mat"][conv], o["beta_mat"][conv], floor=1e-9)) < TOL
    assert np.nanmax(rel_err(np.sqrt(g["beta_var_mat"][conv]), np.sqrt(o["beta_var_mat"][conv]))) < TOL


def test_fit_beta_divergence_sentinel(engine):
    """test_optim.R:29-39 on the engine: the 0/1000 row must report iter == maxit."""
    y = np.array([[0, 0, 0, 0, 0, 1000, 1000, 0, 0, 0], [5, 7, 6, 4, 5, 9, 11, 8, 10, 12]], dtype=np.int32)
    x = np.c_[np.ones(10), np.r_[np.zeros(5), np.ones(5)]]
    r = engine.fitBeta(y, x, np.ones((2, 10)), [0.1, 0.1], [1, 0], np.ones((2, 2)), np.full(2, 1e-6) / np.log(2) ** 2,
                       None, False, 1e-8, 100, True, 0.5)
    assert r["iter"][0] == 100 and r["iter"][1] < 100


def test_fit_beta_weight_zero_equals_dropped_sample(engine):
    c = make_case(200, 10, seed=73)
    alpha = np.clip(0.1 + 4 / c["baseMean"], 1e-8, 10)
    w = np.ones(c["counts"].shape)
    w[:, 0] = 0.0
    a = engine.fitBeta(**beta_args(c, alpha, weights=w, useWeights=True))
    sub = dict(c)
    sub["counts"], sub["nf"], sub["x"] = c["counts"][:, 1:], c["nf"][:, 1:], c["x"][1:]
    b = engine.fitBeta(**beta_args(sub, alpha))
    assert np.allclose(a["beta_mat"], b["beta_mat"], atol=1e-8)
    assert np.allclose(a["beta_var_mat"], b["beta_var_mat"], rtol=1e-7)
    assert np.allclose(a["deviance"], b["deviance"], rtol=1e-9)


# ---------------------------------------------------------------- full-size properties (BASELINE.json config 2)

def test_c2_full_size_properties(engine, oracle):
    """50k x 100 is too slow to check gene by gene against the oracle in a test; use size-independent properties:
    chunked == whole, restart-from-optimum is a fixed point, maxit=0 reproduces the covariance block, and an
    oracle spot check on a random 1% of the genes."""
    c = make_case(50000, 100, seed=20260923 + 2)
    n = len(c["counts"])
    a = disp_args(c, c["mu"], np.log(c["alpha0"]))
    g = engine.fitDisp(**a)
    # chunked == whole (bitwise: genes are independent and the kernels are deterministic)
    sl = slice(12345, 13345)
    sub = {k: (v[sl] if isinstance(v, np.ndarray) and v.shape[:1] == (n,) else v) for k, v in a.items()}
    gs = engine.fitDisp(**sub)
    for k in DISP_KEYS + ("iter", "iter_accept"):
        assert np.array_equal(gs[k], g[k][sl]), k
    # restart from the optimum with a tiny tolerance: the first accepted step must already satisfy change < tol
    conv = (g["iter"] < 100) & (g["log_alpha"] > np.log(1e-7))
    a2 = disp_args(c, c["mu"], g["log_alpha"])
    g2 = engine.fitDisp(**a2)
    assert np.max(np.abs(g2["log_alpha"][conv] - g["log_alpha"][conv])) < 5e-2
    assert np.all(g2["last_lp"][conv] >= g["last_lp"][conv] - 1e-6 * (1 + np.abs(g["last_lp"][conv])))
    # oracle spot check
    rng = np.random.default_rng(0)
    idx = np.sort(rng.choice(n, 500, replace=False))
    subo = {k: (v[idx] if isinstance(v, np.ndarray) and v.shape[:1] == (n,) else v) for k, v in a.items()}
    o = oracle.fitDisp(**subo, with_margin=True)
    gsub = {k: v[idx] for k, v in g.items()}
    _compare_disp(gsub, o, "c2 spot check")
    # fitBeta: maxit = 0 from the fitted coefficients reproduces variance / hat diagonal / contrast
    alpha = np.clip(np.exp(g["log_alpha"]), 1e-8, 100)
    fb = engine.fitBeta(**beta_args(c, alpha))
    fb0 = engine.fitBeta(**beta_args(c, alpha, beta0=fb["beta_mat"], maxit=0))
    for k in ("beta_var_mat", "hat_diagonals", "contrast_num", "contrast_denom"):
        assert np.nanmax(rel_err(fb0[k], fb[k], floor=1e-12)) < 1e-9, k
    # hat diagonals sum to the effective number of parameters (trace of the hat matrix <= p)
    tr = fb["hat_diagonals"].sum(axis=1)
    ok = fb["iter"] < 100
    assert np.all(tr[ok] <= 2 + 1e-9) and np.median(tr[ok]) > 1.99


# ---------------------------------------------------------------- general p (5 <= p <= 32): shared-memory path

def _mu_from_fit(oracle, c, x, alpha, lam=None, beta0=None):
    fit = oracle.fitBeta(**beta_args(c, alpha, x=x, lam=lam, beta0=beta0))
    return np.maximum(c["nf"] * np.exp(fit["beta_mat"] @ x.T), 0.5)


@pytest.mark.parametrize("kind,seed", [("factor10", 81), ("expanded11", 82), ("covariates7", 83)])
def test_general_p_parity(engine, oracle, kind, seed, n=400):
    """BASELINE.json config 4 shapes (10-level factor: p=10 MLE pass, 11-column expanded matrix with ridge) and a
    design with continuous covariates (> 32 distinct rows -> samplewise normal equations)."""
    from deseq2_b200 import synth
    rng = np.random.default_rng(seed)
    m = 60
    if kind == "factor10":
        x = synth.design_factor(m, 10)
        lam = np.full(10, 1e-6) / np.log(2) ** 2
    elif kind == "expanded11":
        x = synth.design_factor_expanded(m, 10)
        lam = np.r_[1e-6, np.full(10, 1.0 / 0.7)] / np.log(2) ** 2
    else:
        x = np.c_[synth.design_batch_condition(m, 3), rng.normal(0, 1, (m, 3))]
        lam = np.full(7, 1e-6) / np.log(2) ** 2
    p = x.shape[1]
    xgen = synth.design_factor(m, 10) if kind == "expanded11" else x
    c = make_case(n, m, x=xgen, seed=seed, betaSD=0.5)
    c["x"] = x
    n = len(c["counts"])
    if kind == "expanded11":
        beta0 = np.zeros((n, p))
        beta0[:, 0] = np.log(c["baseMean"])
    else:
        Q, R = np.linalg.qr(x)
        beta0 = np.linalg.solve(R, Q.T @ np.log(c["counts"] / c["nf"] + 0.1).T).T
    alpha = np.clip(0.1 + 4 / c["baseMean"], 1e-8, m)
    a = beta_args(c, alpha, x=x, lam=lam, beta0=beta0, contrast=np.r_[np.zeros(p - 1), 1.0])
    g, o = engine.fitBeta(**a), oracle.fitBeta(**a)
    _compare_beta(g, o, f"beta/{kind}", tol=2e-6 if kind == "expanded11" else TOL)
    mu = np.maximum(c["nf"] * np.exp(o["beta_mat"] @ x.T), 0.5)
    xd = xgen if kind == "expanded11" else x       # dispersion fits always use the full-rank matrix
    c["x"] = xd
    d = disp_args(c, mu, np.log(c["alpha0"]), prior_mean=np.log(alpha), sigmasq=0.7, usePrior=True)
    _compare_disp(engine.fitDisp(**d), oracle.fitDisp(**d, with_margin=True), f"disp/{kind}", min_robust=0.85)
    w = _weights_for(c, seed)
    d = disp_args(c, mu, np.log(c["alpha0"]), weights=w, useWeights=True)
    _compare_disp(engine.fitDisp(**d), oracle.fitDisp(**d, with_margin=True), f"disp-w/{kind}", min_robust=0.85)
    grid = np.linspace(np.log(1e-8), np.log(m), 20)
    sel = slice(0, 40)
    kw = dict(ySEXP=c["counts"][sel], xSEXP=xd, mu_hatSEXP=mu[sel], disp_gridSEXP=grid,
              log_alpha_prior_meanSEXP=np.log(alpha)[sel], log_alpha_prior_sigmasqSEXP=0.5, usePriorSEXP=True,
              weightsSEXP=None, useWeightsSEXP=False, weightThresholdSEXP=1e-2, useCRSEXP=True)
    gg, og = engine.fitDispGrid(**kw)["log_alpha"], oracle.fitDispGrid(**kw)["log_alpha"]
    assert np.mean(np.abs(gg - og) < 1e-9) > 0.9


@pytest.mark.parametrize("m,G,seed", [(7, 6, 1), (31, 5, 2), (33, 6, 3), (64, 12, 4), (100, 7, 5), (257, 10, 6), (40, 32, 7),
                                      (1000, 10, 8)])
def test_segmented_general_p_kernels(engine, oracle, m, G, seed):
    """The segmented general-p kernels (csrc/fit_generic_seg.cuh: samples sorted by design group, lane chunks, per-lane
    segment sums) on grouped designs of every shape: unequal group sizes in shuffled sample order, m below / across /
    far above the warp width, as many groups as lanes, a genuine (not replicated) normalisation-factor matrix, rows
    with counts beyond 8 and 16 bits (gathered from global memory), double-typed counts.  Checked against the oracle
    and against the kernels of fit_generic.cu (B200NB_GENERIC_SEG=0, read per launch) on the same inputs."""
    import os
    from deseq2_b200 import synth
    rng = np.random.default_rng(900 + seed)
    sizes = rng.multinomial(m - G, rng.dirichlet(np.full(G, 0.7))) + 1      # every group at least one sample
    gid = rng.permutation(np.repeat(np.arange(G), sizes))
    levels = min(G, 6)                                                      # p = levels (+1 covariate-like column)
    x = np.zeros((m, levels))
    x[:, 0] = 1.0
    for k in range(1, levels):
        x[:, k] = (gid % levels == k)
    if G > levels:
        x = np.c_[x, (gid // levels).astype(float)]                         # distinguishes the remaining groups
    assert len(np.unique(x, axis=0)) == G and np.linalg.matrix_rank(x) == x.shape[1]
    p = x.shape[1]
    assert p > 4          # the general-p kernels (p <= 4 runs on the register-resident kernels)
    n = 40 if m >= 1000 else 150
    c = make_case(n, m, x=synth.design_condition(m), seed=seed, betaSD=0.5)
    n = len(c["counts"])
    counts = c["counts"].copy()
    counts[0] = np.minimum(counts[0] * 0 + rng.integers(300, 5000, m), 2 ** 31 - 1)    # beyond 8 bits
    counts[1] = rng.integers(70000, 400000, m)                                          # beyond 16 bits
    c["counts"] = counts
    c["x"] = x
    nf = c["nf"] * np.exp(rng.normal(0, 0.1, c["nf"].shape))                            # a real matrix
    nf /= np.exp(np.mean(np.log(nf), axis=1, keepdims=True))
    alpha = np.clip(0.1 + 4 / np.maximum(c["baseMean"], 1.0), 1e-8, max(10, m))
    beta0 = np.zeros((n, p))
    beta0[:, 0] = np.log(np.maximum(counts.mean(axis=1), 0.1))
    lam = np.full(p, 1e-6) / np.log(2) ** 2
    for variant in ("nf-matrix", "sf-vector", "f64-counts"):
        a = beta_args(c, alpha, x=x, lam=lam, beta0=beta0, contrast=np.r_[np.zeros(p - 1), 1.0],
                      nf=nf if variant == "nf-matrix" else None,
                      y=counts.astype(np.float64) if variant == "f64-counts" else None)
        g = engine.fitBeta(**a, return_mu=True)
        o = oracle.fitBeta(**a)
        _compare_beta(g, o, f"seg beta {variant} m={m} G={G}")
        os.environ["B200NB_GENERIC_SEG"] = "0"
        try:
            g0 = engine.fitBeta(**a, return_mu=True)
        finally:
            os.environ.pop("B200NB_GENERIC_SEG")
        assert np.array_equal(g["iter"], g0["iter"])
        for k in ("beta_mat", "beta_var_mat", "hat_diagonals", "mu", "deviance"):
            assert np.nanmax(rel_err(g[k], g0[k], floor=1e-9)) < 1e-8, (variant, k)
    mu = np.maximum(nf * np.exp(o["beta_mat"] @ x.T), 0.5)
    for variant in ("mle", "map", "f64-counts, no CR"):
        d = disp_args(c, mu, np.log(c["alpha0"]), prior_mean=np.log(alpha), sigmasq=0.7, usePrior=variant == "map",
                      useCR=variant != "f64-counts, no CR", y=counts.astype(np.float64) if "f64" in variant else None)
        g = engine.fitDisp(**d)
        _compare_disp(g, oracle.fitDisp(**d, with_margin=True), f"seg disp {variant} m={m} G={G}", min_robust=0.7)
        os.environ["B200NB_GENERIC_SEG"] = "0"
        try:
            g0 = engine.fitDisp(**d)
        finally:
            os.environ.pop("B200NB_GENERIC_SEG")
        same = (g["iter"] == g0["iter"]) & (g["iter_accept"] == g0["iter_accept"])
        assert same.mean() > 0.9
        assert np.nanmax(rel_err(g["initial_lp"], g0["initial_lp"])) < 1e-9
        assert np.nanmax(rel_err(g["log_alpha"][same], g0["log_alpha"][same], floor=1e-3)) < 1e-6


def test_generic_kernels_on_small_p_designs():
    """Cross-check: force the general-p (shared-memory) kernels onto the p <= 4 cases above in a fresh process
    (the switch is read once per process) -- both kernel families must agree with the oracle on the same inputs."""
    import os
    import subprocess
    import sys
    if os.environ.get("B200NB_FORCE_GENERIC"):
        pytest.skip("already running with the generic kernels forced")
    env = dict(os.environ, B200NB_FORCE_GENERIC="1")
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(here, "test_parity_gpu.py"), "-q", "-m", "gpu", "-k",
                        "mle_parity or map_parity or fit_beta_parity or weights_and_designs or designs_weights_nf "
                        "or maxit0 or grid_parity or drop_a_design"], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]


# ---------------------------------------------------------------- edge shapes (test_edge_case.R:5-19 analogues)

@pytest.mark.parametrize("n,m", [(1, 4), (3, 5), (7, 33), (2, 3000)])
def test_edge_shapes(engine, oracle, n, m):
    """One gene (test_edge_case.R:5-11), m not a multiple of 4 / 32, a single trip of the sample loop, a very
    long row; intercept-only and two-group designs; an all-zero row passes through without crashing."""
    rng = np.random.default_rng(n * 1000 + m)
    x = np.c_[np.ones(m), (np.arange(m) % 2).astype(float)]
    mu_true = rng.uniform(5, 200, (n, 1)) * np.exp(0.5 * x[:, 1])[None, :]
    y = rng.negative_binomial(5.0, 5.0 / (5.0 + mu_true)).astype(np.int32)
    if n > 2:
        y[-1] = 0                                       # all-zero gene
    mu = np.maximum(mu_true, 0.5)
    la = np.log(np.full(n, 0.2))
    kw = dict(ySEXP=y, xSEXP=x, mu_hatSEXP=mu, log_alphaSEXP=la, log_alpha_prior_meanSEXP=la,
              log_alpha_prior_sigmasqSEXP=1.0, min_log_alphaSEXP=np.log(1e-9), kappa_0SEXP=1.0, tolSEXP=1e-6,
              maxitSEXP=100, usePriorSEXP=False, weightsSEXP=None, useWeightsSEXP=False, weightThresholdSEXP=1e-2,
              useCRSEXP=True)
    g, o = engine.fitDisp(**kw), oracle.fitDisp(**kw, with_margin=True)
    ok = (o["margin"] > ROBUST) & np.isfinite(o["last_lp"])
    assert np.array_equal(g["iter"][ok], o["iter"][ok])
    assert np.all(rel_err(g["log_alpha"][ok], o["log_alpha"][ok], floor=1e-9) < TOL)
    for xx in (x, np.ones((m, 1))):
        p = xx.shape[1]
        kb = dict(ySEXP=y, xSEXP=xx, nfSEXP=np.ones((n, m)), alpha_hatSEXP=np.full(n, 0.2),
                  contrastSEXP=np.r_[1.0, np.zeros(p - 1)], beta_matSEXP=np.tile(np.r_[3.0, np.zeros(p - 1)], (n, 1)),
                  lambdaSEXP=np.full(p, 1e-6) / np.log(2) ** 2, weightsSEXP=None, useWeightsSEXP=False, tolSEXP=1e-8,
                  maxitSEXP=100, useQRSEXP=True, minmuSEXP=0.5)
        gb, ob = engine.fitBeta(**kb), oracle.fitBeta(**kb)
        assert np.array_equal(gb["iter"], ob["iter"])
        assert np.nanmax(rel_err(gb["beta_mat"], ob["beta_mat"], floor=1e-7)) < TOL
        assert np.nanmax(rel_err(gb["hat_diagonals"], ob["hat_diagonals"], floor=1e-9)) < TOL


def test_empty_input_is_a_no_op(engine):
    x = np.c_[np.ones(6), np.r_[0, 0, 0, 1, 1, 1.0]]
    r = engine.fitDisp(np.zeros((0, 6), np.int32), x, np.zeros((0, 6)), np.zeros(0), np.zeros(0), 1.0, -20.0, 1.0, 1e-6,
                       10, False, None, False, 1e-2, True)
    assert r["log_alpha"].shape == (0,)
    b = engine.fitBeta(np.zeros((0, 6), np.int32), x, np.zeros((0, 6)), np.zeros(0), [1, 0], np.zeros((0, 2)),
                       [1e-6, 1e-6], None, False, 1e-8, 10, True, 0.5)
    assert b["beta_mat"].shape == (0, 2)


# ---------------------------------------------------------------- BASELINE.json config shapes (3, 4, 5), spot checks

@pytest.mark.parametrize("name,n,m", [("C3", 1500, 500), ("C4", 400, 1000), ("C5", 1500, 200)])
def test_config_shapes_spot_check(engine, oracle, name, n, m):
    """The sample counts and designs of BASELINE.json configs 3-5 at a reduced gene count (genes are independent, so
    the per-gene arithmetic is the full-size arithmetic): C3 ~batch+condition (3x2, p=4, m=500), C4 10-level factor
    (p=10) plus its 11-column expanded matrix with ridge (m=1000), C5 full ~batch+condition (2x2, p=3) and reduced
    ~batch (p=2) for the LRT (m=200)."""
    from deseq2_b200 import synth
    if name == "C3":
        x = synth.design_batch_condition(m, 3)
        fits = [(x, None)]
    elif name == "C4":
        x = synth.design_factor(m, 10)
        xe = synth.design_factor_expanded(m, 10)
        fits = [(x, None), (xe, np.r_[1e-6, np.full(10, 1.0 / 0.5)] / np.log(2) ** 2)]
    else:
        x = synth.design_batch_condition(m, 2)
        fits = [(x, None), (x[:, :2], None)]
    c = make_case(n, m, x=x, seed={"C3": 303, "C4": 404, "C5": 505}[name], betaSD=0.5)
    alpha = np.clip(0.1 + 4 / c["baseMean"], 1e-8, m)
    betas = None
    for xf, lam in fits:
        p = xf.shape[1]
        if np.linalg.matrix_rank(xf) == p:
            Q, R = np.linalg.qr(xf)
            b0 = np.linalg.solve(R, Q.T @ np.log(c["counts"] / c["nf"] + 0.1).T).T
        else:
            b0 = np.zeros((len(c["counts"]), p))
            b0[:, 0] = np.log(c["baseMean"])
        a = beta_args(c, alpha, x=xf, lam=lam, beta0=b0)
        g, o = engine.fitBeta(**a), oracle.fitBeta(**a)
        _compare_beta(g, o, f"{name} beta p={p}", tol=2e-6 if lam is not None else TOL)
        if betas is None:
            betas = o["beta_mat"]
    mu = np.maximum(c["nf"] * np.exp(betas @ x.T), 0.5)
    d = disp_args(c, mu, np.log(c["alpha0"]))
    gd = engine.fitDisp(**d)
    _compare_disp(gd, oracle.fitDisp(**d, with_margin=True), f"{name} disp mle", min_robust=0.8)
    d2 = disp_args(c, mu, gd["log_alpha"], prior_mean=np.log(alpha), sigmasq=0.5, usePrior=True)
    _compare_disp(engine.fitDisp(**d2), oracle.fitDisp(**d2, with_margin=True), f"{name} disp map", min_robust=0.8)


def test_beta_prior_sequence_engine_vs_oracle(engine, oracle):
    """BASELINE.json config 4's call sequence (betaPrior: MLE fit p=10, prior variance, MAP fit on the 11-column
    expanded matrix) through the same host glue with the CUDA engine and with the oracle."""
    from deseq2_b200 import pipeline, synth
    m, levels = 120, 10
    g = (np.arange(m) * levels) // m
    d = synth.make_example_counts(600, m, x=synth.design_factor(m, levels), seed=61, betaSD=0.8)
    counts = d["counts"][d["counts"].sum(axis=1) > 0]
    sf = d["sizeFactors"]
    nf = np.broadcast_to(sf[None, :], counts.shape)
    bm = (counts / sf).mean(axis=1)
    dispFit = 0.1 + 4 / bm
    disp = np.clip(dispFit, 1e-8, m)
    a = pipeline.fitGLMsWithPrior(counts, nf, [g], disp, bm, dispFit, engine=engine)
    b = pipeline.fitGLMsWithPrior(counts, nf, [g], disp, bm, dispFit, engine=oracle)
    assert np.max(rel_err(a["betaPriorVar"], b["betaPriorVar"])) < 1e-6
    assert np.array_equal(a["fit"]["betaIter"], b["fit"]["betaIter"])
    conv = b["fit"]["betaConv"]
    assert np.max(np.abs(a["fit"]["betaMatrix"][conv] - b["fit"]["betaMatrix"][conv])) < 2e-6
    assert np.max(rel_err(a["fit"]["betaSE"][conv], b["fit"]["betaSE"][conv])) < 2e-6


# ---------------------------------------------------------------- post-rule parity (what DESeq() keeps), every gene

@pytest.mark.parametrize("m,n,max_raw_mismatch", [(4, 3000, 0.25), (6, 3000, 0.20), (8, 3000, 0.15), (12, 3000, 0.08),
                                                  (100, 2000, 0.01)])
def test_post_rule_parity_every_gene(engine, oracle, m, n, max_raw_mismatch):
    """R/core.R:784-848 and :1019-1115 turn fitDisp's raw output into dispGeneEst / dispMAP / dispersion (noIncrease
    rule, clamps, grid refit of unconverged genes); R/fitNbinomGLMs.R:180-235 turns fitBeta's into betaMatrix / betaSE.
    Raw iteration counts may differ on knife-edge genes (most genes of a 3-vs-3 experiment start at alpha = minDisp,
    where the reference's own lgamma(y + 1e8) - lgamma(1e8) is rounding noise), so the raw mismatch rate is printed
    and bounded -- but what DESeq() keeps must agree with the oracle on EVERY gene to 1e-6."""
    from deseq2_b200 import pipeline, synth
    x = synth.design_condition(m)
    d = synth.make_example_counts(n, m, x=x, seed=600 + m)
    counts = d["counts"][d["counts"].sum(axis=1) > 0]
    sf = d["sizeFactors"]
    ge_e = pipeline.estimateDispersionsGeneEst(counts, sf, x, engine=engine)
    ge_o = pipeline.estimateDispersionsGeneEst(counts, sf, x, engine=oracle)
    raw = np.mean((ge_e["dispRes"]["iter"] != ge_o["dispRes"]["iter"])
                  | (ge_e["dispRes"]["iter_accept"] != ge_o["dispRes"]["iter_accept"]))
    print(f"\nm={m}: raw fitDisp (MLE) iter / iter_accept differ from the oracle on {100 * raw:.2f}% of {len(counts)} genes")
    assert raw <= max_raw_mismatch
    e = rel_err(ge_e["dispGeneEst"], ge_o["dispGeneEst"])
    assert np.max(e) < TOL, (np.max(e), int(np.sum(e >= TOL)))
    # the MAP step and the Wald fit from identical (oracle-side) inputs
    tf = pipeline.estimateDispersionsFit(ge_o["dispGeneEst"], ge_o["baseMean"])
    pv = pipeline.estimateDispersionsPriorVar(tf["varLogDispEsts"], m, 2, ge_o["dispGeneEst"], tf["dispFit"])
    a = (counts, x, ge_o["mu"], ge_o["dispGeneEst"], tf["dispFit"], pv, tf["varLogDispEsts"])
    mp_e, mp_o = pipeline.estimateDispersionsMAP(*a, engine=engine), pipeline.estimateDispersionsMAP(*a, engine=oracle)
    rawm = np.mean(mp_e["dispRes"]["iter"] != mp_o["dispRes"]["iter"])
    print(f"m={m}: raw fitDisp (MAP) iter differs on {100 * rawm:.2f}% of the genes")
    assert rawm <= max_raw_mismatch
    for k in ("dispMAP", "dispersion"):
        e = rel_err(mp_e[k], mp_o[k])
        assert np.max(e) < TOL, (k, np.max(e), int(np.sum(e >= TOL)))
    assert np.array_equal(mp_e["dispOutlier"], mp_o["dispOutlier"])
    nf = np.broadcast_to(sf[None, :], counts.shape)
    fe = pipeline.fitNbinomGLMs(counts, nf, x, mp_o["dispersion"], engine=engine, useOptim=False)
    fo = pipeline.fitNbinomGLMs(counts, nf, x, mp_o["dispersion"], engine=oracle, useOptim=False)
    assert np.array_equal(fe["betaIter"], fo["betaIter"]) and np.array_equal(fe["betaConv"], fo["betaConv"])
    conv = fo["betaConv"]
    assert np.max(rel_err(fe["betaMatrix"][conv], fo["betaMatrix"][conv], floor=1e-6)) < TOL
    assert np.max(rel_err(fe["betaSE"][conv], fo["betaSE"][conv])) < TOL
    assert np.max(rel_err(fe["logLike"][conv], fo["logLike"][conv])) < TOL


# ---------------------------------------------------------------- host-path input cache (content-addressed) and speculation

def _host_stats():
    import ctypes as C
    import deseq2_b200
    st = (C.c_longlong * 6)()
    deseq2_b200.lib().b200nb_host_stats(st, 6)
    return dict(h2d=st[0], d2h=st[1], hits=st[2], misses=st[3], hit_bytes=st[4], hashed=st[5])


def test_host_cache_is_content_addressed_and_never_stale(engine, oracle):
    """The host entry points keep device copies of their input matrices keyed by CONTENT.  (1) a fresh copy of the same
    matrix at another address is a hit (no upload) with identical results; (2) the same buffer modified IN PLACE in a
    few entries far from the sampled fingerprint blocks must NOT be served from the cache -- the speculative launch is
    discarded and the results are those of the modified data; (3) a normalisation-factor matrix that is a replicated
    size-factor vector except for one entry deep inside takes the matrix path; (4) b200nb_cache_clear forgets."""
    import deseq2_b200
    L = deseq2_b200.lib()
    c = make_case(3000, 40, seed=77)
    a = disp_args(c, c["mu"], np.log(c["alpha0"]))
    L.b200nb_cache_clear()
    s0 = _host_stats()
    g1 = engine.fitDisp(**a)
    s1 = _host_stats()
    assert s1["misses"] - s0["misses"] == 2 and s1["h2d"] - s0["h2d"] > c["counts"].size * 12
    a2 = dict(a, ySEXP=np.array(c["counts"], copy=True), mu_hatSEXP=np.array(c["mu"], copy=True))   # new addresses
    g2 = engine.fitDisp(**a2)
    s2 = _host_stats()
    assert s2["hits"] - s1["hits"] == 2 and s2["h2d"] - s1["h2d"] < 0.2 * c["counts"].size * 12
    for k in DISP_KEYS + ("iter", "iter_accept"):
        assert np.array_equal(g1[k], g2[k], equal_nan=True), k
    # (2) in-place change of two entries in the middle of the buffers
    y3 = np.asfortranarray(a2["ySEXP"])
    mu3 = np.asfortranarray(a2["mu_hatSEXP"])
    y3[1501, 17] += 40
    mu3[1502, 23] *= 3.0
    a3 = dict(a, ySEXP=y3, mu_hatSEXP=mu3)
    g3 = engine.fitDisp(**a3)
    o3 = oracle.fitDisp(**a3, with_margin=True)
    for gene in (1501, 1502):
        assert g3["log_alpha"][gene] != g1["log_alpha"][gene]
        assert abs(g3["initial_lp"][gene] - o3["initial_lp"][gene]) < 1e-9 * abs(o3["initial_lp"][gene])
    other = np.ones(len(y3), bool)
    other[[1501, 1502]] = False
    assert np.array_equal(g3["log_alpha"][other], g1["log_alpha"][other])
    # (3) nf: replicated size factors except one entry that none of the probed rows sees
    alpha = np.clip(0.1 + 4.0 / c["baseMean"], 1e-8, 10)
    b = beta_args(c, alpha)
    r_vec = engine.fitBeta(**b)
    nf2 = np.array(c["nf"], copy=True)
    nf2[777, 5] *= 1.5
    r_mat = engine.fitBeta(**beta_args(c, alpha, nf=nf2))
    o_mat = oracle.fitBeta(**beta_args(c, alpha, nf=nf2))
    assert np.max(rel_err(r_mat["beta_mat"], o_mat["beta_mat"], floor=1e-8)) < TOL
    assert abs(r_mat["beta_mat"][777, 0] - r_vec["beta_mat"][777, 0]) > 1e-6
    rest = np.arange(len(alpha)) != 777
    assert np.max(rel_err(r_mat["beta_mat"][rest], r_vec["beta_mat"][rest], floor=1e-8)) < 1e-9
    # (4) clear: the next call uploads again -- here in 3 row chunks whose kernels overlap the next chunk's upload
    # (the default for >= 16384 genes); bit-identical to the single-piece call, and the chunk-wise uploaded copy is a
    # valid cache entry afterwards (its content hash is computed on the device from the assembled copy)
    import os
    L.b200nb_cache_clear()
    s4 = _host_stats()
    os.environ["B200NB_CHUNKS"] = "3"
    try:
        g5 = engine.fitDisp(**a)
    finally:
        del os.environ["B200NB_CHUNKS"]
    s5 = _host_stats()
    assert s5["misses"] - s4["misses"] == 2
    for k in DISP_KEYS + ("iter", "iter_accept"):
        assert np.array_equal(g5[k], g1[k], equal_nan=True), k
    g6 = engine.fitDisp(**a2)
    s6 = _host_stats()
    assert s6["hits"] - s5["hits"] == 2
    for k in DISP_KEYS + ("iter", "iter_accept"):
        assert np.array_equal(g6[k], g1[k], equal_nan=True), k
