"""The argument contract of the C ABI (include/b200nb.h), checked the same way for every device entry point: one valid
call succeeds, and each class of bad argument that applies to the entry point -- an unknown y_type, a row stride below
m, a NULL y, a NULL output it must write, an element size other than 4 or 8 -- is refused with a message before
anything is launched.  Runs the engine's CUDA source on the SIMT emulator (`emu` fixture), where device pointers are
host pointers.  Also: the host entry points refuse an unknown y_type, and the ctypes signatures of deseq2_b200/_lib.py
match the header's parameter lists."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, M, P, LD, T = 4, 4, 1, 4, 2          # genes, samples, design columns, row stride, filter thresholds


def _buffers():
    """Small inputs that every entry point accepts, as numpy arrays (kept alive by the dict)."""
    rng = np.random.default_rng(3)
    f64 = lambda *sh: np.zeros(sh, dtype=np.float64)
    b = {
        "y": (rng.integers(1, 20, (N, LD))).astype(np.int32), "x": np.ones((P, M)), "mu": np.full((N, LD), 5.0),
        "sf": np.ones(M), "nf": np.ones((N, LD)), "proj": np.full((P, M), 1.0 / M), "la": np.full(N, -1.0),
        "vec_n": np.full(N, 0.1), "contrast": np.ones(P), "beta": np.full((P, N), 1.0), "lam": np.full(P, 1e-6),
        "grid": np.linspace(np.log(1e-8), np.log(10.0), 20), "hat": np.full((N, LD), 0.25), "w": np.ones((N, LD)),
        "cell_ptr": np.array([0, M], dtype=np.int32), "cell_samples": np.arange(M, dtype=np.int32),
        "col_a": np.array([0], dtype=np.int32), "col_b": np.array([-1], dtype=np.int32), "par": f64(M),
        "mask": np.ones(M, dtype=np.int32), "rows": np.array([0], dtype=np.int64), "theta": np.array([0.0, 0.5]),
        "p_sorted": np.linspace(0.01, 0.5, N), "filter": np.linspace(1.0, 4.0, N),
        "order": np.arange(N, dtype=np.int64), "cutoffs": np.array([0.0, 2.0]),
    }
    for k in ("o1", "o2", "o3", "o4", "o5", "o6", "o7", "o8", "o9", "gm", "cm"):
        b[k] = f64(N * LD + 2 * M + 8)
    for k in ("i1", "i2", "i3", "status"):
        b[k] = np.zeros(N * LD, dtype=np.int32)
    return b


def _calls(b):
    """entry point -> (arguments in header order as (name, value) pairs, the bad-argument classes that apply)."""
    P_ = lambda k: C.c_void_p(b[k].ctypes.data)
    yt = ("y", P_("y")), ("y_type", 0)
    dims = ("n", N), ("m", M), ("p", P), ("ld", LD)
    return {
        "b200nb_fit_disp_dev": ([*yt, ("x", P_("x")), ("mu", P_("mu")), ("la", P_("la")), ("pm", P_("la")),
                                 ("s2", 1.0), ("min_la", -20.0), ("k0", 1.0), ("tol", 1e-6), ("maxit", 10),
                                 ("prior", 0), ("w", None), ("use_w", 0), ("wt", 1e-2), ("cr", 1), *dims,
                                 ("out", P_("o1")), ("it", P_("i1")), ("ia", P_("i2")), ("o2", P_("o2")),
                                 ("o3", P_("o3")), ("o4", P_("o4")), ("o5", P_("o5")), ("o6", P_("o6")),
                                 ("o7", P_("o7")), ("stream", None)], ("y_type", "ld", "y", "out")),
        "b200nb_fit_disp_grid_dev": ([*yt, ("x", P_("x")), ("mu", P_("mu")), ("grid", P_("grid")), ("ng", 20),
                                      ("pm", P_("la")), ("s2", 1.0), ("prior", 0), ("w", None), ("use_w", 0),
                                      ("wt", 1e-2), ("cr", 1), *dims, ("out", P_("o1")), ("stream", None)],
                                     ("y_type", "ld", "y", "out")),
        "b200nb_fit_beta_dev": ([*yt, ("x", P_("x")), ("nf", P_("sf")), ("nf_vec", 1), ("alpha", P_("vec_n")),
                                 ("contrast", P_("contrast")), ("beta", P_("beta")), ("lam", P_("lam")), ("w", None),
                                 ("use_w", 0), ("tol", 1e-8), ("maxit", 10), ("qr", 1), ("minmu", 0.5), *dims,
                                 ("out", P_("o1")), ("var", P_("o2")), ("iter", P_("o3")), ("hat", None),
                                 ("cn", P_("o4")), ("cd", P_("o5")), ("dev", P_("o6")), ("mu", None),
                                 ("stream", None)], ("y_type", "ld", "y", "out")),
        "b200nb_nb_loglik_dev": ([*yt, ("x", P_("x")), ("nf", P_("sf")), ("nf_vec", 1), ("alpha", P_("vec_n")),
                                  ("beta", P_("beta")), ("w", None), ("use_w", 0), ("minmu", 0.0), *dims,
                                  ("out", P_("o1")), ("mu", None), ("stream", None)], ("y_type", "ld", "y", "out")),
        "b200nb_beta_optim_dev": ([*yt, ("x", P_("x")), ("nf", P_("sf")), ("nf_vec", 1), ("alpha", P_("vec_n")),
                                   ("lam", P_("lam")), ("beta", P_("beta")), ("w", None), ("use_w", 0), ("maxit", 10),
                                   *dims, ("out", P_("o1")), ("conv", P_("i1")), ("iter", P_("i2")),
                                   ("stream", None)], ("y_type", "ld", "y", "out")),
        "b200nb_to_gene_major_dev": ([("src", P_("mu")), ("out", P_("o1")), ("n", N), ("m", M), ("ld", LD),
                                      ("elem_size", 8), ("stream", None)], ("ld", "out", "elem_size")),
        "b200nb_to_col_major_dev": ([("src", P_("mu")), ("out", P_("o1")), ("n", N), ("m", M), ("ld", LD),
                                     ("stream", None)], ("ld", "out")),
        **{name: ([*yt, ("x", P_("x")), ("proj", P_("proj")), ("factors", P_(fac)), ("xim", 1.0),
                   ("min_disp", 1e-8), ("max_disp", 10.0), ("minmu", 0.5), *dims, ("out", P_("o1")),
                   ("base_var", P_("o2")), ("all_zero", P_("i1")), ("alpha0", P_("o3")), ("mu_lin", extra_mu),
                   ("beta0", P_("o5")), *extra, ("stream", None)], ("y_type", "ld", "y", "out"))
           for name, fac, extra_mu, extra in (
               ("b200nb_prep_dev", "sf", P_("o4"), ()),
               ("b200nb_prep_nf_dev", "nf", P_("o4"), ()),
               ("b200nb_prep_weighted_dev", "sf", None, (("w", P_("w")), ("wt", 1e-2), ("wn", P_("o6")),
                                                        ("wf", P_("i2")), ("status", P_("status")))))},
        "b200nb_trend_fit_dev": ([("means", P_("filter")), ("disps", P_("vec_n")), ("n", N), ("min_disp", 1e-8),
                                  ("out", P_("o1")), ("stream", None)], ("out",)),
        **{name: ([*yt, ("mu", P_("mu")), ("hat", P_("hat")), ("factors", P_(fac)), ("cell_ptr", P_("cell_ptr")),
                   ("cell_samples", P_("cell_samples")), ("ncell", 1), *dims, ("cooks", P_("o1")),
                   ("out", P_("o2")), ("robust", P_("o3")), ("stream", None)], ("y_type", "ld", "y", "out"))
           for name, fac in (("b200nb_cooks_dev", "sf"), ("b200nb_cooks_nf_dev", "nf"))},
        **{name: ([*yt, *divisor, ("poscounts", 0), ("n", N), ("m", M), ("ld", LD), ("lg", P_("o1")),
                   ("gm", P_("gm")), ("cm", P_("cm")), ("out", P_("o2")), ("nfin", P_("i1")), ("stream", None)],
                  ("y_type", "ld", "y", "out"))
           for name, divisor in (("b200nb_size_factors_dev", ()),
                                 ("b200nb_size_factors_norm_dev", (("divisor", P_("nf")),)))},
        "b200nb_beta_prior_quantile_dev": ([("beta", P_("beta")), ("n", N), ("p", P), ("bm", P_("filter")),
                                            ("df", P_("vec_n")), ("col_a", P_("col_a")), ("col_b", P_("col_b")),
                                            ("k", 1), ("prob", 0.95), ("out", P_("o1")), ("stream", None)], ("out",)),
        "b200nb_sf_iterate_objective_dev": ([*yt, ("q", P_("mu")), ("alpha", P_("vec_n")), ("par", P_("par")),
                                             ("h", 1e-3), ("Q", 0.05), ("n", N), ("m", M), ("ld", LD),
                                             ("tile", 0), ("out", P_("o1")), ("stream", None)],
                                            ("y_type", "ld", "y", "out")),
        "b200nb_transform_dev": ([*yt, ("sf", P_("sf")), ("nf", None), ("n", N), ("m", M), ("ld", LD),
                                  ("mode", 0), ("c0", 0.05), ("c1", 2.0), ("out", P_("o1")), ("ld_out", M),
                                  ("stream", None)], ("y_type", "ld", "ld_out", "y", "out")),
        "b200nb_rlog_fit_dev": ([*yt, ("sf", P_("sf")), ("nf", None), ("intercept", None), ("disp", P_("vec_n")),
                                 ("n", N), ("m", M), ("ld", LD), ("bpv", 1.0), ("tol", 1e-4), ("maxit", 10),
                                 ("minmu", 0.5), ("out", P_("o1")), ("ld_out", M), ("icpt", P_("o2")),
                                 ("iter", P_("o3")), ("stream", None)], ("y_type", "ld", "ld_out", "y", "out")),
        "b200nb_rlog_prior_var_dev": ([*yt, ("sf", P_("sf")), ("nf", None), ("bm", P_("filter")),
                                       ("disp", P_("vec_n")), ("n", N), ("m", M), ("ld", LD), ("out", P_("o1")),
                                       ("stream", None)], ("y_type", "ld", "y", "out")),
        "b200nb_results_gene_dev": ([*yt, ("n", N), ("m", M), ("ld", LD), ("lfc", P_("vec_n")), ("se", P_("filter")),
                                     ("stat", P_("vec_n")), ("pv", P_("p_sorted")), ("negate", 0),
                                     ("mask", P_("mask")), ("lrt", 0), ("alt", 0), ("T", 0.0), ("max_cooks", None),
                                     ("cutoff", 0.0), ("keep", None), ("replace", None), ("bm", None),
                                     ("out", P_("o1")), ("o2", P_("o2")), ("o3", P_("o3")), ("o4", P_("o4")),
                                     ("stream", None)], ("y_type", "ld", "y", "out")),
        "b200nb_results_heuristic_dev": ([*yt, ("rows", P_("rows")), ("k", 1), ("m", M), ("ld", LD),
                                          ("cooks", P_("hat")), ("ld_cooks", LD), ("out", P_("i1")),
                                          ("stream", None)], ("y_type", "ld", "ld_cooks", "y", "out")),
        "b200nb_filter_cutoffs_dev": ([("filter", P_("filter")), ("n", N), ("theta", P_("theta")), ("t", T),
                                       ("out", P_("o1")), ("stream", None)], ("out",)),
        "b200nb_filter_numrej_dev": ([("p", P_("p_sorted")), ("f", P_("filter")), ("n", N), ("c", P_("cutoffs")),
                                      ("t", T), ("method", 0), ("alpha", 0.1), ("out", P_("i1")), ("stream", None)],
                                     ("out",)),
        "b200nb_padj_dev": ([("p", P_("p_sorted")), ("f", P_("filter")), ("order", P_("order")), ("n", N),
                             ("cutoffs", None), ("j", 0), ("method", 0), ("out", P_("o1")), ("stream", None)],
                            ("out",)),
    }


_BAD = {"y_type": {"y_type": 2}, "ld": {"ld": M - 1}, "ld_out": {"ld_out": M - 1}, "ld_cooks": {"ld_cooks": M - 1},
        "y": {"y": None}, "out": {"out": None}, "elem_size": {"elem_size": 2}}


def test_every_device_entry_point_is_covered():
    from deseq2_b200 import _lib
    assert sorted(_calls(_buffers())) == sorted(s for s in _lib.SIGNATURES if s.endswith("_dev"))


@pytest.mark.parametrize("name", sorted(_calls(_buffers())))
def test_device_entry_point_argument_contract(emu, name):
    from deseq2_b200 import _lib
    L = _lib.lib()
    b = _buffers()
    args, classes = _calls(b)[name]
    fn = getattr(L, name)
    call = lambda **kw: fn(*[kw.get(k, v) for k, v in args])
    assert call() == 0, (name, L.b200nb_last_error())
    for cls in classes:
        launches = L.b200nb_kernel_launches()
        assert call(**_BAD[cls]) != 0, (name, cls)
        assert L.b200nb_last_error(), (name, cls)
        assert L.b200nb_kernel_launches() == launches, (name, cls)


def test_host_entry_points_refuse_unknown_y_type(emu):
    """Refused before any device call (the host entry points would otherwise pick the upload element size from it)."""
    from deseq2_b200 import _lib
    L = _lib.lib()
    y, x, v = np.ones((N, M), dtype=np.int32), np.ones((M, P)), np.zeros(N * M)
    o = [np.zeros(N * M) for _ in range(9)]
    Pv = lambda a: C.c_void_p(a.ctypes.data)
    outs = [Pv(a) for a in o]
    rc = L.b200nb_fit_disp(Pv(y), 2, Pv(x), Pv(v), Pv(v), Pv(v), 1.0, -20.0, 1.0, 1e-6, 10, 0, None, 0, 1e-2, 1, N, M, P,
                           *outs)
    assert rc != 0 and b"y_type" in L.b200nb_last_error()
    rc = L.b200nb_fit_disp_grid(Pv(y), 2, Pv(x), Pv(v), Pv(np.linspace(-18, 2, 20)), 20, Pv(v), 1.0, 0, None, 0, 1e-2,
                                1, N, M, P, outs[0])
    assert rc != 0 and b"y_type" in L.b200nb_last_error()
    rc = L.b200nb_fit_beta(Pv(y), 2, Pv(x), Pv(np.ones(N * M)), Pv(v), Pv(np.ones(P)), Pv(v), Pv(np.ones(P)), None, 0,
                           1e-8, 10, 1, 0.5, N, M, P, *outs[:8])
    assert rc != 0 and b"y_type" in L.b200nb_last_error()


def _header_params():
    """symbol -> parameter kinds ("ptr", "int", "long long", "double", "size_t") from include/b200nb.h."""
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200nb.h")).read(), flags=re.S)
    out = {}
    for name, params in re.findall(r"\b(b200nb_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt):
        kinds = []
        for prm in (q.strip() for q in params.split(",")):
            if prm in ("", "void"):
                continue
            if "*" in prm:
                kinds.append("ptr")
            else:
                kinds.append(next(k for k in ("long long", "double", "size_t", "int") if re.match(k + r"\b", prm)))
        out[name] = kinds
    return out


def test_ctypes_signatures_match_header():
    from deseq2_b200 import _lib
    kind = {C.c_int: "int", C.c_longlong: "long long", C.c_double: "double", C.c_size_t: "size_t",
            C.c_void_p: "ptr"}
    hdr = _header_params()
    assert sorted(hdr) == sorted(_lib.SIGNATURES)
    for name, argt in _lib.SIGNATURES.items():
        got = ["ptr" if hasattr(t, "contents") else kind[t] for t in argt]
        assert got == hdr[name], name
