"""The indicator-design variants of the small-p fit kernels, bit for bit against the general variants.

Each small-p kernel (fit_disp_kernel, fit_disp_grp_kernel, fit_beta_kernel, fit_beta_grp_kernel) is compiled twice:
a general variant and one for 0/1 indicator designs (smallp.cuh::indicator_design: column 0 all 1.0, every other entry
+0.0 or 1.0), which forms no FP64 design products and takes the (a, a) sums from the (a, 0) sums.  Both are launched;
the one that does not fit the design returns after the design test.  The indicator variant promises the general
variant's results bit for bit.

The comparator is the design's twin: every +0.0 of columns 1 .. p-1 becomes -0.0.  The twin never passes the design
test, so it runs the general variant, and it changes no value the general variant computes (every product with -0.0
is a signed zero, and adding -0.0 to a sum that starts at +0.0 leaves it unchanged).  So X and its twin, fitted in one
process on one build, must agree byte for byte on every output, NaN bits included.  Each case also goes against the
CPU oracle, so that both variants cannot be wrong together.

  * every instantiation (kernel family, P, USE_W, lanes per gene) of the small-p launchers, for fitDisp (MLE, MAP, no
    Cox-Reid), fitDispGrid (no variant: a control) and fitBeta (maxit 100 / 0, size-factor vector / nf matrix), through
    the host C ABI and the device entry points; a coverage test reads the emulator's launch log to confirm each case
    lands on the instantiation it is meant for;
  * which variant does the work, per design, from the number of warp collectives the emulator counted per launch: a
    variant that returns after the design test executes exactly one __all_sync per thread;
  * degenerate indicator designs (an all-zero column, duplicated columns, weights that remove a column), where NaN and
    inf positions must agree too;
  * b200nb_kernel_launches() against the emulator's own count of launches, for every entry point run here.

The emulated half runs on every CPU run (about 40 seconds on one core, measured with
`pytest tests/test_indicator_designs.py -m "not gpu"`); the bit-identity and oracle cases run again on the H100 under
-m gpu, where they check the compiled SASS of each pair."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

from helpers import beta_args, disp_args, make_case, rel_err
from test_parity_gpu import _compare_beta, _compare_disp, _weights_for
from test_sample_counts import LANES_8, LONG_ROWS, _emu_lib, backend, grp16_last, launch_log, smallp_last  # noqa: F401

N_GENES = 4          # a TAB, a BIG and a GEN gene, and one whose weights remove a design column
WEIGHT_THRESHOLD = 1e-2


# ---------------------------------------------------------------- designs

def x_intercept(m):
    return np.ones((m, 1))


def x_condition(m):
    return np.c_[np.ones(m), np.r_[np.zeros((m + 1) // 2), np.ones(m // 2)]]


def x_batch(n_batch):
    def f(m):
        from deseq2_b200 import synth
        return synth.design_batch_condition(m, n_batch)     # p = n_batch + 1
    return f


def x_a_times_b(m):
    """~a * b, two two-level factors: [1, a, b, a:b]; the interaction column is the AND of columns 1 and 2."""
    a = (np.arange(m) % 2).astype(float)
    b = ((np.arange(m) // 2) % 2).astype(float)
    return np.c_[np.ones(m), a, b, a * b]


# ~1, ~condition, ~batch + condition with 2 and 3 batches, ~a * b
DESIGNS = {"intercept": x_intercept, "condition": x_condition, "batch2": x_batch(2), "batch3": x_batch(3),
           "axb": x_a_times_b}


def twin(x):
    """Every +0.0 of columns 1 .. p-1 as -0.0: the same values, but the design test fails, so the general variant runs."""
    t = np.array(x, dtype=np.float64, copy=True)
    sub = t[:, 1:]
    sub[(sub == 0.0) & ~np.signbit(sub)] = -0.0
    return t


def _bits(v):
    return np.array([v], dtype=np.uint64).view(np.float64)[0]


# ---------------------------------------------------------------- the cases of section 1
# (design, m, weights, nf, counts dtype).  Lanes per gene: m <= LANES_8 runs the 8-lane kernels, above that the 16-lane
# kernels up to grp16_last, then the one-warp kernel; the 32-lane cases take the first m past both fitDisp's and
# fitBeta's last 16-lane m, so that every family runs its 32-lane kernel.

def _m32(p, w, nf):
    return max(grp16_last("disp", p, w), grp16_last("beta", p, w, nf == "sf")) + 1


def _cases():
    cs = []
    spec = [
        # 8 lanes per gene
        ("intercept", 40, False, "sf", "i4"), ("intercept", 18, True, "matrix", "f8"),
        ("condition", LANES_8, False, "sf", "i4"), ("condition", 23, True, "matrix", "f8"),
        ("batch2", 30, False, "matrix", "f8"), ("batch2", LANES_8, True, "sf", "i4"),
        ("batch3", LANES_8, False, "sf", "i4"), ("axb", 37, True, "matrix", "f8"),
        # 16 lanes per gene
        ("intercept", LANES_8 + 1, False, "matrix", "i4"), ("intercept", 90, True, "sf", "f8"),
        ("condition", 66, False, "matrix", "f8"), ("condition", LANES_8 + 1, True, "sf", "i4"),
        ("batch2", LANES_8 + 1, False, "sf", "i4"), ("batch2", 101, True, "matrix", "f8"),
        ("axb", LANES_8 + 1, False, "sf", "f8"), ("batch3", 66, True, "matrix", "i4"),
        # 32 lanes per gene (one warp)
        ("intercept", _m32(1, False, "matrix"), False, "matrix", "i4"), ("intercept", _m32(1, True, "matrix"), True, "matrix", "f8"),
        ("condition", _m32(2, False, "sf"), False, "sf", "i4"), ("condition", _m32(2, True, "matrix"), True, "matrix", "f8"),
        ("batch2", _m32(3, False, "matrix"), False, "matrix", "f8"),
        ("batch2", _m32(3, True, "sf"), True, "sf", "i4"),
        ("batch3", _m32(4, False, "matrix"), False, "matrix", "i4"),
        ("axb", _m32(4, True, "matrix"), True, "matrix", "f8"),
    ]
    for design, m, w, nf, dt in spec:
        assert m <= smallp_last("disp", 4, True) and m <= smallp_last("beta", 4, True, False)
        cs.append((f"{design}-m{m}{'-w' if w else ''}-{nf}-{dt}", design, m, w, nf, dt))
    return cs


CASES = _cases()


def _counts(x, dt, seed, n=N_GENES):
    """n genes of NB counts on design x: gene 0 in TAB mode (integral, max < 256), gene 1 in BIG mode (min >= 10, max
    >= 256), gene 2 in GEN mode (a zero and a count >= 256); f8 counts also get fractions (GEN)."""
    m = x.shape[0]
    c = make_case(n, m, x=x, seed=seed, betaSD=0.5, drop_zero=False)
    y = np.array(c["counts"], dtype=np.float64)
    rng = np.random.default_rng(seed)
    y[0] = np.minimum(y[0], 255.0)
    y[1] = np.maximum(y[1], 10.0)
    y[1, rng.integers(m)] = 300.0
    y[2, rng.integers(m)] = 0.0
    y[2, rng.integers(m)] = 400.0
    if n > 3:
        y[3, 0] = max(y[3, 0], 1.0)
    if dt == "f8":
        y[2:, rng.integers(m, size=3)] += 0.5
        c["counts"] = y
    else:
        c["counts"] = y.astype(np.int32)
    return c


def _inputs(design, m, weights, nf, dt, oracle, n=N_GENES, x=None):
    x = DESIGNS[design](m) if x is None else x
    seed = 1000 + m
    c = _counts(x, dt, seed, n)
    c["x"] = x
    rng = np.random.default_rng(seed + 1)
    if nf == "matrix":
        nfm = c["nf"] * np.exp(rng.normal(0, 0.1, c["nf"].shape))
        c["nf"] = nfm / np.exp(np.mean(np.log(nfm), axis=1, keepdims=True))
    c["w"] = None
    if weights:
        w = _weights_for(c, seed)                       # includes values below the Cox-Reid weight threshold
        w[rng.random(w.shape) < 0.05] = 0.0             # and exact zeros
        w[:, 0] = 1.0
        if x.shape[1] > 1 and n > 3:
            # gene 3: every kept row of the last column is zero -> that column is inert (fit_disp.cu, USE_W)
            w[3, x[:, -1] != 0] = WEIGHT_THRESHOLD / 2
        c["w"] = w
    mean = np.maximum(c["counts"], 0).mean(axis=1) + 1.0
    c["alpha"] = np.clip(0.1 + 4.0 / mean, 1e-8, max(10, m))
    c["alpha0"] = np.clip(c["alpha"] * 1.5, 1e-8, max(10, m))
    Q, R = np.linalg.qr(x)
    c["beta0"] = np.linalg.solve(R, Q.T @ np.log(c["counts"] / c["nf"] + 0.1).T).T
    fit = oracle.fitBeta(**beta_args(c, c["alpha"], weights=c["w"], useWeights=weights))
    c["mu"] = np.maximum(c["nf"] * np.exp(np.nan_to_num(fit["beta_mat"]) @ x.T), 0.5)
    return c


# ---------------------------------------------------------------- runs of every entry point, with the launch counter

class _Counter:
    """On the emulator: b200nb_kernel_launches() must move by exactly the number of launches the emulator ran."""

    def __init__(self, lib):
        self.lib = lib
        if lib is not None:
            lib.simt_emu_launches.restype = C.c_longlong
            lib.b200nb_kernel_launches.restype = C.c_longlong

    @contextlib.contextmanager
    def __call__(self, what):
        if self.lib is None:
            yield
            return
        k0, e0 = self.lib.b200nb_kernel_launches(), self.lib.simt_emu_launches()
        yield
        dk, de = self.lib.b200nb_kernel_launches() - k0, self.lib.simt_emu_launches() - e0
        assert dk == de, f"{what}: b200nb_kernel_launches() counted {dk} launches, the emulator ran {de}"


@contextlib.contextmanager
def _small_p_rows(m, weights):
    """The device entry points send unweighted calls with m >= LONG_ROWS to the segmented kernels (capi.cu::long_rows);
    B200NB_LONG_ROWS=0 keeps them on the small-p kernels."""
    if m < LONG_ROWS or weights:
        yield
        return
    saved = os.environ.get("B200NB_LONG_ROWS")
    os.environ["B200NB_LONG_ROWS"] = "0"
    try:
        yield
    finally:
        if saved is None:
            os.environ.pop("B200NB_LONG_ROWS")
        else:
            os.environ["B200NB_LONG_ROWS"] = saved


def _grid(m):
    return np.linspace(np.log(1e-8), np.log(max(10, m)), 20)


def _args(c):
    """Keyword arguments of every host call, as R passes them."""
    w, uw = c["w"], c["w"] is not None
    p = c["x"].shape[1]
    la0, pm = np.log(c["alpha0"]), np.log(c["alpha"])
    return {
        "mle": disp_args(c, c["mu"], la0, weights=w, useWeights=uw),
        "map": disp_args(c, c["mu"], la0, prior_mean=pm, sigmasq=0.6, usePrior=True, weights=w, useWeights=uw),
        "nocr": disp_args(c, c["mu"], la0, weights=w, useWeights=uw, useCR=False),
        "grid": dict(ySEXP=c["counts"], xSEXP=c["x"], mu_hatSEXP=c["mu"], disp_gridSEXP=_grid(c["x"].shape[0]),
                     log_alpha_prior_meanSEXP=pm, log_alpha_prior_sigmasqSEXP=0.6, usePriorSEXP=True, weightsSEXP=w,
                     useWeightsSEXP=uw, weightThresholdSEXP=WEIGHT_THRESHOLD, useCRSEXP=True),
        "beta": beta_args(c, c["alpha"], weights=w, useWeights=uw),
        # maxit = 0 from the oracle's optimum, contrast on the last column
        "beta0": beta_args(c, c["alpha"], beta0=c["beta_opt"], maxit=0, weights=w, useWeights=uw,
                           contrast=np.r_[np.zeros(p - 1), 1.0]),
    }


def _host_runs(W, c, count):
    a = _args(c)
    res = {}
    for k in ("mle", "map", "nocr"):
        with count(f"host fitDisp {k}"):
            res[k] = W.fitDisp(**a[k])
    with count("host fitDispGrid"):
        res["grid"] = W.fitDispGrid(**a["grid"])
    for k in ("beta", "beta0"):
        with count(f"host fitBeta {k}"):
            res[k] = W.fitBeta(**a[k], return_mu=True)
    return res, a


def _device_runs(D, dev, c, nf, count):
    import torch
    T = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=dev)
    y, mu = D.to_gene_major(c["counts"], dev), D.to_gene_major(c["mu"], dev)
    w = D.to_gene_major(c["w"], dev) if c["w"] is not None else None
    x = c["x"]
    m, p = x.shape
    la0, pm = T(np.log(c["alpha0"])), T(np.log(c["alpha"]))
    host = lambda r: {k: (v.cpu().numpy() if v is not None else None) for k, v in r.items()}
    lmin = float(np.log(1e-8 / 10))
    res = {}
    with _small_p_rows(m, w is not None):
        for k, prior, cr in (("mle", False, True), ("map", True, True), ("nocr", False, False)):
            with count(f"device fit_disp {k}"):
                res[k] = host(D.fit_disp(y, x, mu, la0, pm if prior else la0, 0.6 if prior else 1.0, lmin, 1.0, 1e-6,
                                         100, prior, weights=w, useCR=cr))
        with count("device fit_disp_grid"):
            res["grid"] = host(D.fit_disp_grid(y, x, mu, _grid(m), pm, 0.6, True, weights=w))
        nfd = T(c["sf"]) if nf == "sf" else D.to_gene_major(c["nf"], dev)
        lam = T(np.full(p, 1e-6) / np.log(2) ** 2)
        for k, beta0, maxit, contrast in (("beta", c["beta0"], 100, np.r_[1.0, np.zeros(p - 1)]),
                                          ("beta0", c["beta_opt"], 0, np.r_[np.zeros(p - 1), 1.0])):
            with count(f"device fit_beta {k}"):
                r = host(D.fit_beta(y, x, nfd, T(c["alpha"]), T(contrast), T(beta0.T), lam, 1e-8, maxit, weights=w))
            r["beta_mat"], r["beta_var_mat"] = r["beta_mat"].T, r["beta_var_mat"].T
            # (n, ld) rows: the padding beyond m is never written
            r["hat_diagonals"], r["mu"] = r["hat_diagonals"][:, :m], r["mu"][:, :m]
            r["contrast_num"], r["contrast_denom"] = r["contrast_num"][:, None], r["contrast_denom"][:, None]
            res[k] = r
    return res


def _runs(W, D, dev, lib, c, nf):
    count = _Counter(lib)
    res, args = _host_runs(W, c, count)
    return res, args, _device_runs(D, dev, c, nf, count)


# ---------------------------------------------------------------- checks

def _same_bytes(a, b, name):
    """Every output of run a equals run b byte for byte (NaN payloads and signed zeros included)."""
    assert a.keys() == b.keys(), name
    for call in a:
        assert a[call].keys() == b[call].keys(), (name, call)
        for k in a[call]:
            u, v = a[call][k], b[call][k]
            if u is None or v is None:
                assert u is None and v is None, (name, call, k)
                continue
            u, v = np.ascontiguousarray(u), np.ascontiguousarray(v)
            assert u.dtype == v.dtype and u.shape == v.shape, (name, call, k)
            diff = (u.view(np.uint8) != v.view(np.uint8)).reshape(u.size, -1).any(axis=1) if u.size else []
            bad = np.flatnonzero(diff)
            assert bad.size == 0, (f"{name} {call}: {k} differs in {bad.size} of {u.size} entries, first at flat index "
                                   f"{bad[0]}: {u.reshape(-1)[bad[0]]!r} against {v.reshape(-1)[bad[0]]!r}")


def _check_oracle(res, args, oracle, name):
    for k in ("mle", "map", "nocr"):
        o = oracle.fitDisp(**args[k], with_margin=True)
        g = res[k]
        _compare_disp(g, o, f"{name} {k}", min_robust=0.0)
        # a gene that took the oracle's steps (same iter and iter_accept) is held to 1e-6 even below ROBUST
        same = (g["iter"] == o["iter"]) & (g["iter_accept"] == o["iter_accept"])
        assert same.mean() >= 0.5, f"{name} {k}: only {same.sum()} of {same.size} genes on the oracle's path"
        for key in ("log_alpha", "last_lp", "initial_lp"):
            assert np.max(rel_err(g[key][same], o[key][same])) < 1e-6, (name, k, key)
    og = oracle.fitDispGrid(**args["grid"])["log_alpha"]
    grid = args["grid"]["disp_gridSEXP"]
    d = np.abs(res["grid"]["log_alpha"] - og)
    assert np.max(d) < 2.0 * (grid[1] - grid[0]) / 9.5 and np.mean(d < 1e-9) >= 0.5, f"{name} grid: {d}"
    ob = oracle.fitBeta(**args["beta"])
    _compare_beta(res["beta"], ob, f"{name} beta")
    r0 = res["beta0"]
    assert np.all(r0["iter"] == 0)
    _compare_beta(r0, oracle.fitBeta(**args["beta0"]), f"{name} beta maxit=0")


def _prepare(case, oracle, n=N_GENES):
    name, design, m, weights, nf, dt = case
    c = _inputs(design, m, weights, nf, dt, oracle, n=n)
    if nf == "sf":
        c["nf"] = np.broadcast_to(c["sf"][None, :], c["counts"].shape).copy()
    c["beta_opt"] = oracle.fitBeta(**beta_args(c, c["alpha"], weights=c["w"], useWeights=weights))["beta_mat"]
    return c


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_indicator_variant_matches_its_twin(backend, oracle, case):
    """Section 1: X (indicator variant) and its twin (general variant) agree byte for byte through both entry routes,
    and X agrees with the oracle.  ~1 has no column to flip: oracle only."""
    name, design, m, weights, nf, dt = case
    W, D, dev, lib = backend
    c = _prepare(case, oracle)
    res, args, dres = _runs(W, D, dev, lib, c, nf)
    _check_oracle(res, args, oracle, f"{name} host")
    _check_oracle(dres, args, oracle, f"{name} device")
    if c["x"].shape[1] == 1:
        return
    t = dict(c, x=twin(c["x"]))
    tres, _, tdres = _runs(W, D, dev, lib, t, nf)
    _same_bytes(res, tres, f"{name} host twin")
    _same_bytes(dres, tdres, f"{name} device twin")


# ---------------------------------------------------------------- which instantiation each case reaches (emulator)

def _fit_launches(log):
    """The small-p fit kernel launches of an emulator launch log, in launch order: (kind, P, USE_W, lanes per gene,
    collectives).  The launching function's signature carries the template arguments (launch_disp_grp / launch_beta_grp:
    8 or 16 lanes; launch_disp_t / launch_beta_t: the one-warp kernel, whose fitDispGrid kernel `kg` has no variant and
    is left out, as are classify_kernel and bucket_sort_kernel)."""
    import re
    out = []
    for line in log.splitlines():
        f = [s.strip() for s in line.split(" | ")]
        if len(f) < 5:
            continue
        what, where, coll = f[0], f[1], int(f[4])
        fam = re.search(r"launch_(disp|beta)_(grp|t)\(", where)
        if fam is None or what in ("classify_kernel", "bucket_sort_kernel") or (fam.group(2) == "t" and what == "kg"):
            continue
        p = int(re.search(r"int P = (\d+)", where).group(1))
        w = re.search(r"bool USE_W = (true|false)", where).group(1) == "true"
        gl = re.search(r"int GL = (\d+)", where)
        out.append((fam.group(1), p, w, int(gl.group(1)) if gl else 32, coll))
    return out


def test_cases_cover_every_small_p_instantiation(oracle):
    """Every (kernel family, P, USE_W, lanes per gene) of the small-p launchers is run by some case of section 1, read
    from the emulator's launch log of each case's runs through every entry point."""
    import torch
    from deseq2_b200 import _lib, device as D, wrappers as W
    lib = _emu_lib()
    seen = set()
    saved, saved_stream = _lib._lib, D._stream
    _lib._lib, D._stream = lib, (lambda: C.c_void_p(0))
    try:
        launch_log(lib)
        for case in CASES:
            c = _prepare(case, oracle)
            _runs(W, D, torch.device("cpu"), None, c, case[4])
            seen |= {f[:4] for f in _fit_launches(launch_log(lib))}
    finally:
        _lib._lib, D._stream = saved, saved_stream
    want = {(k, p, w, gl) for k in ("disp", "beta") for p in (1, 2, 3, 4) for w in (False, True)
            for gl in (8, 16, 32)}
    assert want <= seen, f"not reached: {sorted(want - seen)}"


# ---------------------------------------------------------------- which variant does the work (emulator)

def _simple_case(x, n=2, seed=5, weights=None):
    """n genes of NB counts (mean 20) with a flat fitted mean: enough for every entry point to run on any design,
    including singular ones, without an oracle fit."""
    m, p = x.shape
    rng = np.random.default_rng(seed)
    y = rng.negative_binomial(5, 0.2, size=(n, m)).astype(np.int32)
    y[:, 0] = np.maximum(y[:, 0], 1)
    sf = np.exp(rng.normal(0, 0.2, m))
    beta0 = np.zeros((n, p))
    beta0[:, 0] = np.log(np.maximum(y.mean(axis=1), 1.0))
    return {"counts": y, "x": x, "sf": sf, "nf": np.broadcast_to(sf[None, :], (n, m)).copy(),
            "mu": np.maximum(np.exp(beta0[:, :1]) * sf[None, :], 0.5), "alpha0": np.full(n, 0.3),
            "alpha": np.full(n, 0.2), "beta0": beta0, "beta_opt": beta0, "w": weights}


def _emulated():
    """Binds the emulated engine for the duration of a with-block; yields (wrappers, device module, emulator)."""
    @contextlib.contextmanager
    def bound():
        from deseq2_b200 import _lib, device as D, wrappers as W
        lib = _emu_lib()
        saved, saved_stream = _lib._lib, D._stream
        _lib._lib, D._stream = lib, (lambda: C.c_void_p(0))
        launch_log(lib)
        try:
            yield W, D, lib
        finally:
            _lib._lib, D._stream = saved, saved_stream
    return bound()


def _run_and_classify(x, name):
    """Every entry point on design x through both routes; for each small-p fit call, the variant that did the work.
    The launchers launch the general variant first and the indicator variant second (`for (int ind = 0; ind < 2;
    ...)`); the variant that does not fit the design returns after the design test's one __all_sync."""
    import torch
    with _emulated() as (W, D, lib):
        out = _runs(W, D, torch.device("cpu"), lib, _simple_case(x), "sf")
        fl = _fit_launches(launch_log(lib))
    assert fl and len(fl) % 2 == 0, f"{name}: {len(fl)} fit launches, expected pairs"
    kinds = set()
    for gen, ind in zip(fl[0::2], fl[1::2]):
        assert gen[:4] == ind[:4], f"{name}: unpaired launches {gen} {ind}"
        worked = (gen[4] > 1, ind[4] > 1)
        assert sum(worked) == 1 and min(gen[4], ind[4]) == 1, f"{name}: collectives {gen[4]}, {ind[4]} in {gen[:4]}"
        kinds.add("indicator" if worked[1] else "general")
    assert len(kinds) == 1, f"{name}: calls on one design took different variants"
    return kinds.pop(), out


def _with(x, idx, v):
    x = np.array(x, dtype=np.float64, order="F", copy=True)
    x.reshape(-1, order="F")[idx] = v
    return x


def _variant_designs():
    cond = x_condition(12)
    c12 = cond[:, 1]
    ind = {
        "condition": cond, "batch3": x_batch(3)(12), "axb": x_a_times_b(12), "intercept": x_intercept(12),
        "unused-level": np.c_[cond, np.zeros(12)], "duplicated": np.c_[cond, c12], "second-ones": np.c_[cond, np.ones(12)],
        "m2": x_condition(2), "m3": x_condition(3), "m33": x_condition(33), "m65": x_condition(65),
    }
    gen = {f"twin-{k}": twin(v) for k, v in ind.items() if v.shape[1] > 1}
    m = 37                                           # not a multiple of 32: the last entry is in a partial sweep
    base = x_batch(2)(m)                             # p = 3
    P = base.shape[1]
    gen["~0+condition"] = np.c_[1.0 - x_condition(m)[:, 1], x_condition(m)[:, 1]]
    for label, v in (("col0-zero", 0.0), ("col0-negzero", -0.0)):
        for where, idx in (("first", 0), ("last", m - 1)):          # the first and last entry of column 0
            gen[f"{label}-{where}"] = _with(base, idx, v)
    for label, v in (("1+2^-52", _bits(0x3FF0000000000001)), ("0x3FF00000FFFFFFFF", _bits(0x3FF00000FFFFFFFF)),
                     ("dosage-2", 2.0), ("sum-coding-minus1", -1.0), ("half", 0.5), ("subnormal", _bits(1))):
        for where, idx in (("first", 0), ("last", P * m - 1)):
            gen[f"{label}-{where}"] = _with(base, idx, v)
    return ind, gen


IND_DESIGNS, GEN_DESIGNS = _variant_designs()


@pytest.mark.parametrize("name", sorted(IND_DESIGNS))
def test_indicator_designs_take_the_indicator_variant(oracle, name):
    assert _run_and_classify(IND_DESIGNS[name], name)[0] == "indicator"


@pytest.mark.parametrize("name", sorted(GEN_DESIGNS))
def test_other_designs_take_the_general_variant(oracle, name):
    x = GEN_DESIGNS[name]
    kind, out = _run_and_classify(x, name)
    assert kind == "general"
    hi = np.asarray(x, dtype=np.float64).reshape(-1, order="F").view(np.uint64) >> np.uint64(32)
    dev = np.flatnonzero((hi == 0x3FF00000) & (np.asarray(x).reshape(-1, order="F") != 1.0))
    if dev.size:
        # the deviant shares the high word of 1.0: the same design with a -0.0 elsewhere takes the general variant
        # whatever the design test reads, so the two must agree bit for bit -- a test of high words alone would send
        # this design down the indicator path
        z = np.flatnonzero((np.asarray(x)[:, 1:].reshape(-1, order="F") == 0.0)) + x.shape[0]
        y = _with(x, int(z[z != dev[0]][0]), -0.0)
        kind2, out2 = _run_and_classify(y, name + " + -0.0")
        assert kind2 == "general"
        _same_bytes(out[0], out2[0], f"{name} host against the same design with a -0.0")
        _same_bytes(out[2], out2[2], f"{name} device against the same design with a -0.0")


# ---------------------------------------------------------------- degenerate indicator designs

def _degenerate(kind):
    m = 24
    cond = x_condition(m)
    if kind == "zero-column":            # singular X'WX: log(det) fallback, NaN hat diagonals
        return np.c_[cond, np.zeros(m)], None
    if kind == "duplicated-columns":
        return np.c_[cond, cond[:, 1]], None
    w = np.ones((3, m))                  # weights that zero every kept row of the condition column
    w[:, cond[:, 1] != 0] = 0.0
    w[0, 3] = 0.5
    return cond, w


@pytest.mark.parametrize("kind", ["zero-column", "duplicated-columns", "weights-remove-a-column"])
def test_degenerate_indicator_designs(backend, oracle, kind):
    """Both variants agree byte for byte on singular indicator designs, NaN and inf positions and iter included; where
    the oracle defines an output (a finite value or a NaN), the kernels match it."""
    W, D, dev, lib = backend
    x, w = _degenerate(kind)
    c = _simple_case(x, n=3, weights=w)
    res, args, dres = _runs(W, D, dev, lib, c, "sf")
    tres, _, tdres = _runs(W, D, dev, lib, dict(c, x=twin(x)), "sf")
    _same_bytes(res, tres, f"{kind} host twin")
    _same_bytes(dres, tdres, f"{kind} device twin")
    for r, route in ((res, "host"), (dres, "device")):
        for call in ("beta", "beta0"):
            o = oracle.fitBeta(**args[call])
            # beta_mat is left out: along the singular direction only the 1e-6 ridge pins it, so it follows the
            # iteration's rounding (1e-5 apart from the oracle); every other output is determined
            for k in ("beta_var_mat", "hat_diagonals", "contrast_num", "contrast_denom", "deviance"):
                g, ok = np.asarray(r[call][k]), np.asarray(o[k])
                assert np.array_equal(np.isnan(g), np.isnan(ok)), (kind, route, call, k, "NaN positions")
                fin = np.isfinite(ok) & np.isfinite(g)
                assert np.all(rel_err(g[fin], ok[fin], floor=1e-8) < 1e-6), (kind, route, call, k)
