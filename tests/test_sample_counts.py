"""fitDisp / fitDispGrid / fitBeta at every sample count where a launch plan changes, against the CPU oracle.

DESeq2 puts no limit on the number of samples; the fit kernels keep per-sample rows in shared memory and size them
from m, so each launch plan switches route at some m.  Every case here sits on one side of such a switch, derived
below from the plan code (each helper names the line it mirrors), and runs every entry point -- fitDisp MLE and MAP,
fitDispGrid, fitBeta with maxit = 100 and maxit = 0 -- through the host C ABI (wrappers: what the R shim calls) and
through the device entry points (deseq2_b200.device), which route differently (capi.cu::long_rows applies to device
calls only).  Acceptance is test_parity_gpu's: exact iter / iter_accept where the oracle's decision margin is above
ROBUST, 1e-6 relative on every float output, the same final posterior on knife-edge genes.

Each case runs on the SIMT-emulated engine on every CPU run (backend "emu": the product's CUDA sources compiled by
g++, tests/simt_emu/, which refuses launches the H100 refuses) and again on the H100 under -m gpu (backend "gpu").
On the emulator, each pair of cases on both sides of a switch also checks, from the emulator's launch log, that the
route really changes there: if a constant in the plan code moves, that check fails and names the pair.

n is a handful of genes so that m can be large.  CPU run time of the emulated half: about 3 minutes on one core
(measured with `pytest tests/test_sample_counts.py -m "not gpu"`)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from helpers import DEV, beta_args, disp_args, make_case, rel_err
from test_parity_gpu import _compare_beta, _compare_disp, _weights_for

HERE = os.path.dirname(os.path.abspath(__file__))
SMEM = 227 * 1024            # the per-block shared-memory budget every fit plan sizes against
N_GENES = 6


# ---------------------------------------------------------------- the switch points, mirrored from the plan code

def _mpad(m, a):
    return (m + a - 1) & ~(a - 1)


def _last(pred, lo, hi):
    """Largest m in [lo, hi] with pred(m), for pred true at lo and false at hi (monotone)."""
    assert pred(lo) and not pred(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if pred(mid) else (lo, mid)
    return lo


def _disp_smallp(m, p, w):
    """fit_disp.cu::disp_smem: (design bytes, bytes per warp or lane group)."""
    mp = _mpad(m, 4)
    return p * mp * 8, ((3 if w else 2) * mp + 256) * 8


def _beta_smallp(m, p, w, nfvec):
    """fit_beta.cu::beta_smem."""
    mp = _mpad(m, 4)
    return (p + 1) * mp * 8, (2 + (0 if nfvec else 1) + (1 if w else 0)) * mp * 8


# fit_disp_grp.cuh::group_lanes_disp / fit_beta_grp.cuh::group_lanes_beta: `m <= 40 ? 8 : 16`
LANES_8 = 40
# capi.cu::long_rows: `thr = 400; ... m >= thr`
LONG_ROWS = 400
# capi.cu::prepare_design: `with_seg = grouped && m <= 65535` (16-bit sample positions of SegLayout)
SEG_MAX_M = 65535


def grp16_last(kind, p, w, nfvec=True):
    """Last m on the 16-lane kernels: fit_disp.cu::launch_disp_grp / fit_beta.cu::launch_beta_grp,
    `if (gsmem > 227 * 1024 / GrpShape<GL>::ctas) return` with GrpShape<16> = 256 threads, 2 CTAs: 16 lane groups."""
    def fits(m):
        fixed, row = _disp_smallp(m, p, w) if kind == "disp" else _beta_smallp(m, p, w, nfvec)
        return fixed + 16 * row <= SMEM // 2
    return _last(fits, LANES_8 + 1, 100000)


def smallp_last(kind, p, w, nfvec=True):
    """Last m whose one-warp small-p plan fits: fit_disp.cu::fit_disp_smallp_fits / fit_beta.cu::fit_beta_smallp_fits
    (launch_disp_t / launch_beta_t: `if (xbytes + warps * rowbytes > smem_cap)` at one warp)."""
    def fits(m):
        fixed, row = _disp_smallp(m, p, w) if kind == "disp" else _beta_smallp(m, p, w, nfvec)
        return fixed + row <= SMEM - (3104 if kind == "disp" else 5152)   # k{Disp,Beta}SmemCapOneWarp
    return _last(fits, 8, 100000)


def _seg_kmax(gid, G):
    """capi.cu::build_seg_layout: the most group segments any of the 32 lane chunks holds."""
    m = len(gid)
    order = np.argsort(gid, kind="stable")
    q, rem = divmod(m, 32)
    kmax = 1
    for lane in range(32):
        n_l = q + (1 if lane < rem else 0)
        s0 = lane * q + min(lane, rem)
        kmax = max(kmax, len(np.unique(gid[order[s0:s0 + n_l]])) if n_l else 1)
    return kmax


def seg_last(kind, xfun, p, G, nfvec=True):
    """Last m whose segmented plan fits one warp: fit_generic.cu::plan_seg, `if (fixed + warp_bytes > cap)` with
    cap = 227 KB - 4096, fixed / warp_bytes as launch_fit_{disp,beta}_generic compute them (fit_generic_seg.cuh)."""
    ps = p | 1

    def fits(m):
        x = xfun(m)
        gid = np.unique(x, axis=0, return_inverse=True)[1].reshape(-1)
        kmax = _seg_kmax(gid, G)
        mp = _mpad(m, 8)
        seg_tab = (kmax * 32 * 2 + 32 + 2 * G + 15) & ~15
        pair = (p * (p + 1) + 15) & ~15
        Gp = (G + 1) & ~1
        if kind == "disp":
            sat = G == p
            fixed = G * ps * 8 + seg_tab + pair
            warp = 8 * (mp + 3 * kmax * 32 + (0 if sat else 4 * Gp + 4 * p * ps + 32)) + 2 * 1024 + 2 * mp
        else:
            fixed = (G * ps + (2 * mp if nfvec else 0) + 64 + 256) * 8 + seg_tab + pair
            warp = 8 * ((0 if nfvec else 2 * mp) + 2 * kmax * 32 + 5 * Gp + 4 * p * ps + 4 * 32) + 2 * mp
        return fixed + warp <= SMEM - 4096
    return _last(fits, 64, SEG_MAX_M)


def generic_level(kind, m, p, G, grouped, w, nfvec=True):
    """fit_generic.cu::plan: the first rows_global level (0, 1, 2) whose plan_one fits one warp."""
    mp, ps = _mpad(m, 4), p | 1
    if kind == "disp":
        rows, tab, nacc, extra, extra_row = 2 + w, 256, 3, 0, 0
    else:
        rows, tab, nacc, extra, extra_row = (2 if nfvec else 3) + w, 0, 2, 64, mp
    terms, acc = (G, G * 32) if grouped else (mp, mp)
    for level in (0, 1, 2):
        sums = 0 if (level == 2 and not grouped) else nacc * acc + (nacc * terms if grouped else 0) + terms
        warp = (0 if level else rows * mp) + tab + sums + 4 * p * ps + 128
        if level == 2:
            fixed = (G * ps if grouped else 0) + extra
        else:
            fixed = (G if grouped else m) * ps + (m + 1) // 2 + extra + extra_row
        if (fixed + warp) * 8 <= SMEM - 3104:   # plan_one's cap: 227 KB less the static shared memory
            return level
    return None


def generic_last(level, kind, p, G, grouped, w, nfvec=True):
    return _last(lambda m: generic_level(kind, m, p, G, grouped, w, nfvec) <= level, 64, 200000)


# ---------------------------------------------------------------- designs

def x_intercept(m):
    return np.ones((m, 1))


def x_condition(m):
    return np.c_[np.ones(m), np.r_[np.zeros((m + 1) // 2), np.ones(m // 2)]]


def x_batch_condition(m):
    from deseq2_b200 import synth
    return synth.design_batch_condition(m, 3)        # p = 4


def x_factor6(m):
    from deseq2_b200 import synth
    return synth.design_factor(m, 6)                 # p = 6, G = 6: segmented / generic grouped


def x_covariates(m):
    rng = np.random.default_rng(m)
    return np.c_[np.ones(m), rng.normal(0.0, 0.4, (m, 5))]     # p = 6, > 32 distinct rows: generic samplewise


DESIGNS = {"p1": x_intercept, "p2": x_condition, "p4": x_batch_condition, "p6g": x_factor6, "p6c": x_covariates}

# fit_generic_seg.cuh::seg_tab_limit: min(max(2m, 256), kTabSeg = 1024)


def seg_tab_limit(m):
    return min(max(2 * m, 256), 1024)


# ---------------------------------------------------------------- the cases
# (name, design, m, weights, nf, counts dtype).  Pairs that straddle a switch share a name prefix and end in "/lo",
# "/hi"; ROUTE_PAIRS lists them for the route check.

def _cases():
    cs = []

    def pair(name, design, m_lo, w=False, nf="sf", dt="i4"):
        cs.append((f"{name}/lo", design, m_lo, w, nf, dt))
        cs.append((f"{name}/hi", design, m_lo + 1, w, nf, dt))

    # 8 -> 16 lanes per gene (group_lanes_disp / group_lanes_beta)
    pair("lanes", "p2", LANES_8)
    pair("lanes-w", "p2", LANES_8, w=True, nf="matrix")
    # 16-lane kernels -> 32-lane kernel (launch_disp_grp / launch_beta_grp: 227 KB / ctas)
    pair("grp16-disp", "p2", grp16_last("disp", 2, False))
    pair("grp16-disp-w", "p4", grp16_last("disp", 4, True), w=True)
    pair("grp16-beta", "p2", grp16_last("beta", 2, False, True))
    pair("grp16-beta-nf", "p1", grp16_last("beta", 1, False, False), nf="matrix")
    # capi.cu::long_rows (device entry points, unweighted): small-p -> segmented kernels
    pair("long-rows", "p2", LONG_ROWS - 1)
    pair("long-rows-p4", "p4", LONG_ROWS - 1, dt="f8")
    # segmented plan (plan_seg) no longer fits one warp: -> generic grouped kernels
    pair("seg-disp", "p2", seg_last("disp", x_condition, 2, 2))
    pair("seg-beta", "p2", seg_last("beta", x_condition, 2, 2))
    # with_seg: 16-bit sample positions.  The segmented plan stops fitting one warp long before (seg-* above), so both
    # sides run the generic grouped kernels, with and without a segment layout built: not a route pair
    cs.append(("with-seg/at", "p2", SEG_MAX_M, False, "sf", "i4"))
    cs.append(("with-seg/past", "p2", SEG_MAX_M + 1, False, "sf", "i4"))
    # one small-p warp no longer fits (the kernels used to refuse these calls): -> general-p kernels
    pair("smallp-disp", "p2", smallp_last("disp", 2, False))
    pair("smallp-disp-w", "p2", smallp_last("disp", 2, True), w=True)
    pair("smallp-disp-p4-w", "p4", smallp_last("disp", 4, True), w=True, dt="f8")
    pair("smallp-beta", "p2", smallp_last("beta", 2, False, True))
    pair("smallp-beta-nf-w", "p2", smallp_last("beta", 2, True, False), w=True, nf="matrix")
    # plan_one: shared-memory rows -> rows_global = 1 -> rows_global = 2
    for lvl in (0, 1):
        pair(f"rows{lvl}-disp-cov", "p6c", generic_last(lvl, "disp", 6, 0, False, False))
        pair(f"rows{lvl}-beta-cov-w", "p6c", generic_last(lvl, "beta", 6, 0, False, True, False), w=True, nf="matrix")
    pair("rows0-disp-grouped-w", "p6g", generic_last(0, "disp", 6, 6, True, True), w=True)
    pair("rows1-beta-grouped-w", "p6g", generic_last(1, "beta", 6, 6, True, True, True), w=True)
    # well past every switch
    for d in ("p1", "p2", "p4"):
        cs.append((f"far/{d}", d, 20000, False, "sf", "i4"))
        cs.append((f"far/{d}-w", d, 20000, True, "matrix", "f8"))
    cs.append(("far/p6c", "p6c", 10000, False, "sf", "i4"))
    cs.append(("far/p6c-w", "p6c", 10000, True, "matrix", "i4"))
    cs.append(("far/p6g", "p6g", 70000, False, "sf", "i4"))
    return cs


CASES = _cases()
ROUTE_PAIRS = sorted({c[0].rsplit("/", 1)[0] for c in CASES if c[0].endswith(("/lo", "/hi"))})


# ---------------------------------------------------------------- engines

_EMU = {}


def _emu_lib():
    if "lib" not in _EMU:
        sys.path.insert(0, os.path.join(HERE, "simt_emu"))
        import build_emu
        from deseq2_b200 import _lib
        lib = C.CDLL(build_emu.build())
        for name, argt in _lib.SIGNATURES.items():
            f = getattr(lib, name)
            f.argtypes = argt
            f.restype = _lib._RESTYPE.get(name, C.c_int)
        lib.simt_emu_launch_log.restype = C.c_longlong
        lib.simt_emu_launch_log.argtypes = [C.c_char_p, C.c_longlong]
        _EMU["lib"] = lib
    return _EMU["lib"]


def launch_log(lib):
    n = lib.simt_emu_launch_log(None, 0)
    buf = C.create_string_buffer(n + 1)
    lib.simt_emu_launch_log(buf, len(buf))
    return buf.value.decode()


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def backend(request, oracle):
    """(wrappers, device module, torch device, emulator library or None).  The emulated engine is bound for the one
    test only, so that the gpu cases of a full run never see it."""
    import torch
    from deseq2_b200 import _lib, device as D, wrappers
    if request.param == "gpu":
        request.getfixturevalue("engine")
        yield wrappers, D, torch.device(DEV), None
        return
    lib = _emu_lib()
    saved, saved_stream = _lib._lib, D._stream
    _lib._lib, D._stream = lib, (lambda: C.c_void_p(0))
    launch_log(lib)
    try:
        yield wrappers, D, torch.device("cpu"), lib
    finally:
        _lib._lib, D._stream = saved, saved_stream


# ---------------------------------------------------------------- inputs and the runs of every entry point

def _inputs(design, m, weights, nf, dt, seed, n=N_GENES, oracle=None):
    x = DESIGNS[design](m)
    c = make_case(n, m, x=x, seed=seed, betaSD=0.5)
    c["x"] = x
    rng = np.random.default_rng(seed)
    if nf == "matrix":
        nfm = c["nf"] * np.exp(rng.normal(0, 0.1, c["nf"].shape))
        c["nf"] = nfm / np.exp(np.mean(np.log(nfm), axis=1, keepdims=True))
    c["w"] = _weights_for(c, seed) if weights else None
    if dt == "f8":
        c["counts"] = c["counts"].astype(np.float64)
    c["alpha"] = np.clip(0.1 + 4.0 / np.maximum(c["baseMean"], 1.0), 1e-8, max(10, m))
    if c["mu"] is None or nf == "matrix" or weights:
        fit = oracle.fitBeta(**beta_args(c, c["alpha"], weights=c["w"], useWeights=weights))
        c["mu"] = np.maximum(c["nf"] * np.exp(fit["beta_mat"] @ x.T), 0.5)
    return c


def _grid(m):
    return np.linspace(np.log(1e-8), np.log(max(10, m)), 20)


def _host_runs(W, c):
    w, uw = c["w"], c["w"] is not None
    la0 = np.log(c["alpha0"])
    pm = np.log(c["alpha"])
    out = {"mle": disp_args(c, c["mu"], la0, weights=w, useWeights=uw),
           "map": disp_args(c, c["mu"], la0, prior_mean=pm, sigmasq=0.6, usePrior=True, weights=w, useWeights=uw)}
    res = {k: W.fitDisp(**a) for k, a in out.items()}
    m = c["counts"].shape[1]
    gkw = dict(ySEXP=c["counts"], xSEXP=c["x"], mu_hatSEXP=c["mu"], disp_gridSEXP=_grid(m), log_alpha_prior_meanSEXP=pm,
               log_alpha_prior_sigmasqSEXP=0.6, usePriorSEXP=True, weightsSEXP=w, useWeightsSEXP=uw,
               weightThresholdSEXP=1e-2, useCRSEXP=True)
    res["grid"] = W.fitDispGrid(**gkw)
    out["grid"] = gkw
    b = beta_args(c, c["alpha"], weights=w, useWeights=uw)
    res["beta"] = W.fitBeta(**b)
    out["beta"] = b
    b0 = beta_args(c, c["alpha"], beta0=res["beta"]["beta_mat"], maxit=0, weights=w, useWeights=uw,
                   contrast=np.r_[np.zeros(c["x"].shape[1] - 1), 1.0])
    res["beta0"] = W.fitBeta(**b0)
    out["beta0"] = b0
    return res, out


def _device_runs(D, dev, c, nf):
    import torch
    T = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=dev)
    y = D.to_gene_major(c["counts"], dev)
    mu = D.to_gene_major(c["mu"], dev)
    w = D.to_gene_major(c["w"], dev) if c["w"] is not None else None
    m, p = c["x"].shape
    la0, pm = T(np.log(c["alpha0"])), T(np.log(c["alpha"]))
    host = lambda r: {k: (v.cpu().numpy() if v is not None else None) for k, v in r.items()}
    res = {"mle": host(D.fit_disp(y, c["x"], mu, la0, la0, 1.0, float(np.log(1e-8 / 10)), 1.0, 1e-6, 100, False,
                                  weights=w)),
           "map": host(D.fit_disp(y, c["x"], mu, la0, pm, 0.6, float(np.log(1e-8 / 10)), 1.0, 1e-6, 100, True,
                                  weights=w))}
    res["grid"] = host(D.fit_disp_grid(y, c["x"], mu, _grid(m), pm, 0.6, True, weights=w))
    nfd = T(c["sf"]) if nf == "sf" else D.to_gene_major(c["nf"], dev)
    lam = T(np.full(p, 1e-6) / np.log(2) ** 2)

    def beta(beta0, maxit, contrast):
        r = host(D.fit_beta(y, c["x"], nfd, T(c["alpha"]), T(contrast), T(beta0.T), lam, 1e-8, maxit, weights=w))
        r["beta_mat"], r["beta_var_mat"] = r["beta_mat"].T, r["beta_var_mat"].T
        r["hat_diagonals"] = r["hat_diagonals"][:, :m]
        r["contrast_num"], r["contrast_denom"] = r["contrast_num"][:, None], r["contrast_denom"][:, None]   # as R's
        return r
    res["beta"] = beta(c["beta0"], 100, np.r_[1.0, np.zeros(p - 1)])
    res["beta0"] = beta(res["beta"]["beta_mat"], 0, np.r_[np.zeros(p - 1), 1.0])
    return res


def _check_all(res, args, oracle, name, device_beta0_from=None):
    """Returns how many gene fits of fitDisp MLE and MAP took the oracle's steps (checked to 1e-6)."""
    robust = 0
    for k in ("mle", "map"):
        # the rounding bound of a decision grows with m, so at long rows few of a handful of genes are robust: the
        # robust ones must follow the oracle exactly, the others end at the same posterior
        o = oracle.fitDisp(**args[k], with_margin=True)
        g = res[k]
        _compare_disp(g, o, f"{name} {k}", min_robust=0.0)
        # at long rows the rounding bound of a decision is large, so few genes clear ROBUST; a gene that took the
        # oracle's steps anyway (same iter and iter_accept) is held to 1e-6 as well
        same = (g["iter"] == o["iter"]) & (g["iter_accept"] == o["iter_accept"])
        for key in ("log_alpha", "last_lp", "initial_lp"):
            assert not same.any() or np.max(rel_err(g[key][same], o[key][same])) < 1e-6, (name, k, key)
        robust += int(np.sum(same))
    og = oracle.fitDispGrid(**args["grid"])["log_alpha"]
    grid = args["grid"]["disp_gridSEXP"]
    d = np.abs(res["grid"]["log_alpha"] - og)
    # argmax on a grid: the same grid point unless two posterior values tie to rounding
    assert np.max(d) < 2.0 * (grid[1] - grid[0]) / 9.5 and np.mean(d < 1e-9) >= 0.5, f"{name} grid: {d}"
    _compare_beta(res["beta"], oracle.fitBeta(**args["beta"]), f"{name} beta")
    b0 = dict(args["beta0"])
    if device_beta0_from is not None:
        b0["beta_matSEXP"] = device_beta0_from
    r0 = res["beta0"]
    assert np.all(r0["iter"] == 0)
    _compare_beta(r0, oracle.fitBeta(**b0), f"{name} beta maxit=0")
    return robust


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fit_entry_points_at_sample_count(backend, oracle, case):
    name, design, m, weights, nf, dt = case
    W, D, dev, lib = backend
    c = _case(case, oracle)
    res, args = _host_runs(W, c)
    rob = _check_all(res, args, oracle, f"{name} m={m} host")
    dres = _device_runs(D, dev, c, nf)     # "sf": the device call takes the size-factor vector the rows above repeat
    rob += _check_all(dres, args, oracle, f"{name} m={m} device", device_beta0_from=dres["beta"]["beta_mat"])
    # the 1e-6 checks need genes on the oracle's path: at least half of the 4 n fitDisp fits (MLE / MAP, host / device)
    assert rob >= 2 * len(c["counts"]), f"{name}: only {rob} gene fits on the oracle's path"


def _case(case, oracle, n=None):
    name, design, m, weights, nf, dt = case
    kw = {} if n is None else {"n": n}
    c = _inputs(design, m, weights, nf, dt, seed=m % 1000 + 7, oracle=oracle, **kw)
    if nf == "sf":
        c["nf"] = np.broadcast_to(c["sf"][None, :], c["counts"].shape).copy()
    return c


def _route(log):
    """The fit kernels a run launched, by kernel, launching function (with its template arguments) and block size;
    for the general-p kernels also whether the plan filled shared memory (rows_global moves rows out when it would not
    fit, often at the same block size)."""
    keep = ("launch_disp_t", "launch_disp_grp", "launch_beta_t", "launch_beta_grp", "launch_fit_disp_generic",
            "launch_fit_beta_generic", "launch_disp_seg_t", "launch_beta_seg_t")
    out = set()
    for line in log.splitlines():
        what, where, threads, smem = [s.strip() for s in line.split(" | ")][:4]   # the fifth field: collectives
        if any(k in where for k in keep) and what != "classify_kernel" and what != "bucket_sort_kernel":
            out.add((what, where, threads, "generic" in where and int(smem) > SMEM - 16 * 1024))
    return out


@pytest.mark.parametrize("pair", ROUTE_PAIRS)
def test_cases_straddle_a_route_switch(oracle, pair):
    """Each lo/hi pair above must take different launch routes on its two sides, read from the emulator's launch log
    of one gene through every entry point: a pair that no longer does sits beside the switch it is named for, because
    a constant of the plan code moved without the helper that mirrors it."""
    import torch
    from deseq2_b200 import _lib, device as D, wrappers as W
    lib = _emu_lib()
    routes = []
    saved, saved_stream = _lib._lib, D._stream
    _lib._lib, D._stream = lib, (lambda: C.c_void_p(0))
    try:
        for side in ("lo", "hi"):
            case = next(c for c in CASES if c[0] == f"{pair}/{side}")
            c = _case(case, oracle, n=1)
            launch_log(lib)
            _host_runs(W, c)
            _device_runs(D, torch.device("cpu"), c, case[4])
            routes.append(_route(launch_log(lib)))
    finally:
        _lib._lib, D._stream = saved, saved_stream
    assert routes[0] != routes[1], f"{pair}: both sides launch {routes[0]}"


# ---------------------------------------------------------------- count values at a fixed m

def _count_case(design, m, seed, edits, dt="i4"):
    """A case whose gene g has one sample's count set to edits[g] (a boundary value); the other samples stay NB.
    An edit given as ("min", v) sets every count of that gene to at least v instead."""
    x = DESIGNS[design](m)
    c = make_case(len(edits) + 2, m, x=x, seed=seed, betaSD=0.5)
    c["x"] = x
    y = c["counts"].astype(np.float64 if dt == "f8" else np.int64)
    rng = np.random.default_rng(seed)
    for g, e in enumerate(edits):
        if isinstance(e, tuple):
            kind, v = e
            if kind == "min":
                y[g] = np.maximum(y[g], v)
                y[g, rng.integers(m)] = v
                y[g, rng.integers(m)] = 3000           # above every table
            elif kind == "frac":
                y[g, rng.integers(m)] += v
        else:
            y[g, rng.integers(m)] = e
    c["counts"] = y if dt == "f8" else y.astype(np.int32)
    c["alpha"] = np.clip(0.1 + 4.0 / np.maximum(c["baseMean"], 1.0), 1e-8, max(10, m))
    c["w"] = None
    c["mu"] = np.maximum(c["nf"] * np.exp(c["beta0"] @ x.T), 0.5)
    return c


COUNT_CASES = [
    # small-p TAB mode (fit_disp.cu kTabMax = 256) and the generic kTabMaxG = 256: max count 255 / 256; and the IRLS
    # log y! table (nb_logdens.cuh::log_factorial, fit_generic_seg.cuh lfact) at 255 / 256
    ("tab-smallp", "p2", 120, [255, 256], "i4"),
    ("tab-generic", "p6c", 120, [255, 256], "i4"),
    # the segmented factor table: max count seg_tab_limit(m) - 1 / seg_tab_limit(m), hitting its 256, 2m and 1024
    # branches (m = 128, 300, 600)
    *[(f"segtab-m{m}", "p6g", m, [seg_tab_limit(m) - 1, seg_tab_limit(m)], "i4") for m in (128, 300, 600)],
    # the segmented kernels' 16-bit count row against the gather through seg.inv: 65535 / 65536
    ("count16", "p6g", 200, [65535, 65536], "i4"),
    ("count16-long", "p2", 450, [65535, 65536], "i4"),
    # BIG against GEN mode on rows above the table: minimum count 10 / 9
    ("big-gen", "p2", 100, [("min", 10), ("min", 9)], "i4"),
    ("big-gen-generic", "p6c", 100, [("min", 10), ("min", 9)], "i4"),
    # one non-integer count in a row that is otherwise TAB-able
    ("frac", "p2", 60, [("frac", 0.5), 12], "f8"),
    ("frac-seg", "p6g", 60, [("frac", 0.5), 12], "f8"),
]


@pytest.mark.parametrize("case", COUNT_CASES, ids=[c[0] for c in COUNT_CASES])
def test_fit_entry_points_at_count_values(backend, oracle, case):
    name, design, m, edits, dt = case
    W, D, dev, _ = backend
    c = _count_case(design, m, 400 + m, edits, dt)
    res, args = _host_runs(W, c)
    _check_all(res, args, oracle, f"{name} host")
    dres = _device_runs(D, dev, c, "sf")
    _check_all(dres, args, oracle, f"{name} device", device_beta0_from=dres["beta"]["beta_mat"])


# ---------------------------------------------------------------- the other kernels that size shared memory by m
# At the largest sweep m each of these is past its shared-memory plan (launch_prep: one warp above 200 KB near
# m = 8500; launch_cooks likewise; launch_beta_optim above 200 KB near m = 12 800) and takes its global-rows route.
# nb_loglik, rlog_fit, transform and the size-factor kernels use static shared memory only (nothing sized by m): one
# case each shows that they run there too.  The host mirror (pipeline.*) is the reference, as in their own tests.
M_MAX = max(c[2] for c in CASES)


def _far_counts(m, x, seed, n=6):
    from deseq2_b200 import synth
    d = synth.make_example_counts(n, m, x=x, seed=seed, betaSD=0.5)
    keep = d["counts"].sum(axis=1) > 0
    return d["counts"][keep], d["sizeFactors"]


@pytest.mark.parametrize("variant", ["sf", "weighted", "nf"])
@pytest.mark.parametrize("design", ["p2", "p6c"])
def test_prep_kernels_at_largest_m(backend, design, variant):
    from deseq2_b200 import pipeline
    W, D, dev, _ = backend
    from deseq2_b200 import device_pipeline as DP
    m = M_MAX
    x = DESIGNS[design](m)
    counts, sf = _far_counts(m, x, 31)
    rng = np.random.default_rng(4)
    kw, div, w = {}, sf, None
    if variant == "weighted":
        w = rng.uniform(0.2, 1.0, counts.shape)
        kw["weights"] = D.to_gene_major(w, dev)
    elif variant == "nf":
        div = sf[None, :] * np.exp(rng.normal(0, 0.1, counts.shape))
        kw["normalizationFactors"] = D.to_gene_major(div, dev)
        kw["xim"] = float(np.mean(1.0 / div.mean(axis=0)))
    pr = DP.prep(D.to_gene_major(counts, dev), x, sf, **kw)
    mv = pipeline.getBaseMeansAndVariances(counts, div, weights=w)
    assert np.max(rel_err(pr["baseMean"].cpu().numpy(), mv["baseMean"])) < 1e-12
    assert np.max(rel_err(pr["baseVar"].cpu().numpy(), mv["baseVar"])) < 1e-10
    norm = counts / div
    mu = np.maximum(pipeline.linearModelMu(norm, x) * div, 0.5)
    if pr["mu_lin"] is not None:            # the weighted variant returns no linear-model mu
        assert np.max(rel_err(pr["mu_lin"].cpu().numpy()[:, :m], mu)) < 1e-10
    Q, R = np.linalg.qr(x)
    b0 = np.linalg.solve(R, Q.T @ np.log(norm + 0.1).T).T
    assert np.max(np.abs(pr["beta0"].cpu().numpy().T - b0)) < 1e-10
    if variant == "weighted":
        assert np.max(np.abs(pr["weightsNorm"].cpu().numpy()[:, :m] - w / w.max(axis=1, keepdims=True))) == 0
        assert not pr["weightsFail"].cpu().numpy().any()


@pytest.mark.parametrize("variant", ["sf", "nf"])
def test_cooks_kernel_at_largest_m(backend, variant):
    from deseq2_b200 import device_pipeline as DP, pipeline
    W, D, dev, _ = backend
    m = M_MAX
    x = x_condition(m)
    counts, sf = _far_counts(m, x, 32)
    rng = np.random.default_rng(5)
    div = sf if variant == "sf" else sf[None, :] * np.exp(rng.normal(0, 0.1, counts.shape))
    n = len(counts)
    mu = np.maximum((counts / div).mean(axis=1, keepdims=True) * div * rng.uniform(0.8, 1.25, (n, m)), 0.5)
    H = rng.uniform(0.0, 2.0 / m, (n, m))
    kw = {} if variant == "sf" else {"normalizationFactors": D.to_gene_major(div, dev)}
    out = DP.cooks(D.to_gene_major(counts, dev), D.to_gene_major(mu, dev), D.to_gene_major(H, dev), x, sf, **kw)
    assert np.max(rel_err(out["robustDisp"].cpu().numpy(), pipeline.robustMethodOfMomentsDisp(counts, div, x))) < 1e-10
    ref = pipeline.calculateCooksDistance(counts, mu, H, div, x)
    assert np.max(rel_err(out["cooks"].cpu().numpy()[:, :m], ref, floor=1e-12)) < 1e-9
    assert np.max(rel_err(out["maxCooks"].cpu().numpy(), pipeline.recordMaxCooks(x, ref), floor=1e-12)) < 1e-9


def test_loglik_and_optim_at_largest_m(backend, oracle):
    """nb_loglik (no shared memory) against nbinomLogLike; beta_optim (two rows of m in shared memory, global past
    200 KB) started at the IRLS optimum stays there: a stationary point of the same likelihood."""
    import torch
    from deseq2_b200 import pipeline
    W, D, dev, _ = backend
    m = M_MAX
    x = x_condition(m)
    counts, sf = _far_counts(m, x, 33)
    n, p = len(counts), x.shape[1]
    c = {"counts": counts, "x": x, "nf": np.broadcast_to(sf[None, :], counts.shape).copy()}
    alpha = np.full(n, 0.1)
    Q, R = np.linalg.qr(x)
    c["beta0"] = np.linalg.solve(R, Q.T @ np.log(counts / sf + 0.1).T).T
    fit = oracle.fitBeta(**beta_args(c, alpha))
    T = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=dev)
    y = D.to_gene_major(counts, dev)
    ll = D.nb_loglik(y, x, T(sf), T(alpha), T(fit["beta_mat"].T))
    mu = sf[None, :] * np.exp(fit["beta_mat"] @ x.T)
    assert np.max(rel_err(ll["logLike"].cpu().numpy(), pipeline.nbinomLogLike(counts, mu, alpha))) < 1e-10
    lam = np.full(p, 1e-6)
    op = D.beta_optim(y, x, T(sf), T(alpha), T(lam), T(fit["beta_mat"].T))
    assert np.all(op["converged"].cpu().numpy() == 1)
    assert np.max(np.abs(op["beta_mat"].cpu().numpy().T - fit["beta_mat"])) < 1e-6


@pytest.mark.parametrize("kind", ["weights-condition", "covariates"])
def test_deseq_device_past_the_old_small_p_ceiling(backend, kind):
    """DESeq_device(weights=...) on ~condition at m = 20 000 and DESeq_device on a p = 6 covariate design at m = 10 000,
    then results_device, against the host mirror pipeline.DESeq / pipeline.results driving the same engine through
    the C ABI, with test_device_pipeline_matches_host_pipeline's tolerances."""
    from deseq2_b200 import device_pipeline as DP, pipeline
    W, D, dev, _ = backend
    m = 20000 if kind.startswith("weights") else 10000
    x = x_condition(m) if kind.startswith("weights") else x_covariates(m)
    counts, sf = _far_counts(m, x, 34, n=8)
    w = np.random.default_rng(6).uniform(0.3, 1.0, counts.shape) if kind.startswith("weights") else None
    y = D.to_gene_major(counts, dev)
    wd = D.to_gene_major(w, dev) if w is not None else None
    host = pipeline.DESeq(counts, x, sizeFactors=sf, engine=W, useOptim=False, weights=w)
    dv = DP.DESeq_device(y, x, sf, useOptim=False, weights=wd)
    idx = dv["idx"].cpu().numpy()
    same = ((dv["dispGeneIter"].cpu().numpy() == host["dispGeneIter"][idx])
            & (dv["dispIter"].cpu().numpy() == host["dispIter"][idx]))
    assert same.mean() >= 0.75, same
    for k in ("dispGeneEst", "dispMAP", "dispersion"):
        assert np.max(rel_err(dv[k].cpu().numpy()[same], host[k][idx][same])) < 1e-6, k
    conv = (host["betaConv"][idx] == 1) & same
    assert conv.any()
    assert np.max(rel_err(dv["betaMatrix"].cpu().numpy()[conv], host["betaMatrix"][idx][conv], floor=1e-6)) < 1e-6
    assert np.max(rel_err(dv["betaSE"].cpu().numpy()[conv], host["betaSE"][idx][conv])) < 1e-6
    rd = DP.results_device(dv, y, x, **({"weights": wd} if w is not None else {}))
    rh = pipeline.results(host, counts, x, engine=W)
    for k in ("log2FoldChange", "lfcSE", "pvalue"):
        got, ref = rd[k].cpu().numpy()[conv], rh[k][idx][conv]
        assert np.max(rel_err(got, ref, floor=1e-10)) < 1e-5, k
