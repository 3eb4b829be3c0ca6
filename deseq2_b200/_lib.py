"""ctypes loader for libb200nb.so (C ABI: include/b200nb.h).  Fails loudly; never falls back."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.environ.get("B200NB_LIB") or os.path.join(_HERE, "libb200nb.so")   # B200NB_LIB: experiment builds
_lib = None


class EngineError(RuntimeError):
    """Raised when the CUDA engine is missing or a C-ABI call reports failure."""


def lib_path() -> str:
    return _SO


def build(force: bool = False) -> str:
    """Compile csrc/*.cu for sm_90a into deseq2_b200/libb200nb.so (in-tree, nvcc cross-compiles without a GPU)."""
    args = ["make", "-C", os.path.join(_HERE, "csrc"), "-s", "-j4"]
    if force:
        args.append("-B")
    subprocess.check_call(args)
    return _SO


dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int32)
vp = C.c_void_p

# symbol -> argtypes; every symbol declared in include/b200nb.h appears here (tests/test_abi.py checks both ways)
_D, _I, _LL = C.c_double, C.c_int, C.c_longlong
SIGNATURES = {
    "b200nb_fit_disp": [vp, _I, vp, vp, vp, vp, _D, _D, _D, _D, _I, _I, vp, _I, _D, _I, _I, _I, _I] + [vp] * 9,
    "b200nb_fit_disp_grid": [vp, _I, vp, vp, vp, _I, vp, _D, _I, vp, _I, _D, _I, _I, _I, _I, vp],
    "b200nb_fit_beta": [vp, _I, vp, vp, vp, vp, vp, vp, vp, _I, _D, _I, _I, _D, _I, _I, _I] + [vp] * 8,
    "b200nb_fit_disp_dev": [vp, _I, vp, vp, vp, vp, _D, _D, _D, _D, _I, _I, vp, _I, _D, _I, _I, _I, _I, _LL]
    + [vp] * 9 + [vp],
    "b200nb_fit_disp_grid_dev": [vp, _I, vp, vp, vp, _I, vp, _D, _I, vp, _I, _D, _I, _I, _I, _I, _LL, vp, vp],
    "b200nb_fit_beta_dev": [vp, _I, vp, vp, _I, vp, vp, vp, vp, vp, _I, _D, _I, _I, _D, _I, _I, _I, _LL]
    + [vp] * 8 + [vp],
    "b200nb_nb_loglik_dev": [vp, _I, vp, vp, _I, vp, vp, vp, _I, _D, _I, _I, _I, _LL, vp, vp, vp],
    "b200nb_beta_optim_dev": [vp, _I, vp, vp, _I, vp, vp, vp, vp, _I, _I, _I, _I, _I, _LL, vp, vp, vp, vp],
    "b200nb_to_gene_major_dev": [vp, vp, _I, _I, _LL, _I, vp],
    "b200nb_to_col_major_dev": [vp, vp, _I, _I, _LL, vp],
    "b200nb_prep_dev": [vp, _I, vp, vp, vp, _D, _D, _D, _D, _I, _I, _I, _LL, vp, vp, vp, vp, vp, vp, vp],
    "b200nb_prep_weighted_dev": [vp, _I, vp, vp, vp, _D, _D, _D, _D, _I, _I, _I, _LL, vp, vp, vp, vp, vp, vp, vp, _D,
                                 vp, vp, vp, vp],
    "b200nb_prep_nf_dev": [vp, _I, vp, vp, vp, _D, _D, _D, _D, _I, _I, _I, _LL, vp, vp, vp, vp, vp, vp, vp],
    "b200nb_trend_fit_dev": [vp, vp, _I, _D, vp, vp],
    "b200nb_cooks_dev": [vp, _I, vp, vp, vp, vp, vp, _I, _I, _I, _I, _LL, vp, vp, vp, vp],
    "b200nb_cooks_nf_dev": [vp, _I, vp, vp, vp, vp, vp, _I, _I, _I, _I, _LL, vp, vp, vp, vp],
    "b200nb_size_factors_dev": [vp, _I, _I, _I, _I, _LL, vp, vp, vp, vp, vp, vp],
    "b200nb_size_factors_norm_dev": [vp, _I, vp, _I, _I, _I, _LL, vp, vp, vp, vp, vp, vp],
    "b200nb_beta_prior_quantile_dev": [vp, _I, _I, vp, vp, vp, vp, _I, _D, vp, vp],
    "b200nb_sf_iterate_objective_dev": [vp, _I, vp, vp, vp, _D, _D, _I, _I, _LL, _I, vp, vp],
    "b200nb_transform_dev": [vp, _I, vp, vp, _I, _I, _LL, _I, _D, _D, vp, _LL, vp],
    "b200nb_rlog_fit_dev": [vp, _I, vp, vp, vp, vp, _I, _I, _LL, _D, _D, _I, _D, vp, _LL, vp, vp, vp],
    "b200nb_rlog_prior_var_dev": [vp, _I, vp, vp, vp, vp, _I, _I, _LL, vp, vp],
    "b200nb_results_gene_dev": [vp, _I, _I, _I, _LL, vp, vp, vp, vp, _I, vp, _I, _I, _D, vp, _D, vp, vp, vp, vp, vp,
                                vp, vp, vp],
    "b200nb_results_heuristic_dev": [vp, _I, vp, _I, _I, _LL, vp, _LL, vp, vp],
    "b200nb_filter_cutoffs_dev": [vp, _I, vp, _I, vp, vp],
    "b200nb_filter_numrej_dev": [vp, vp, _I, vp, _I, _I, _D, vp, vp],
    "b200nb_padj_dev": [vp, vp, vp, _I, vp, _I, _I, vp, vp],
    "b200nb_last_error": [],
    "b200nb_device_count": [],
    "b200nb_kernel_launches": [],
    "b200nb_release_workspace": [],
    "b200nb_cache_clear": [],
    "b200nb_host_alloc": [C.c_size_t],
    "b200nb_host_free": [vp],
    "b200nb_host_stats": [vp, _I],
    "b200nb_version": [],
    "b200nb_test_special": [vp, _I, vp, vp, vp],
    "b200nb_test_hash": [vp, _LL, _I, _LL, vp],
}
_RESTYPE = {
    "b200nb_last_error": C.c_char_p,
    "b200nb_version": C.c_char_p,
    "b200nb_kernel_launches": C.c_longlong,
    "b200nb_release_workspace": None,
    "b200nb_cache_clear": None,
    "b200nb_host_alloc": C.c_void_p,
    "b200nb_host_free": None,
}


def lib():
    """Return the loaded engine library; raise EngineError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            raise EngineError(
                f"{_SO} not found: the CUDA engine has not been built (run `python -c 'import __graft_entry__ as g; "
                "g.build()'` or `make -C deseq2_b200/csrc`). There is no CPU fallback.")
        try:
            l = C.CDLL(_SO)
        except OSError as e:  # pragma: no cover
            raise EngineError(f"cannot load {_SO}: {e}") from e
        if hasattr(l, "simt_emu_launches") and os.environ.get("B200NB_TEST_EMULATOR") != "1":
            # tests/simt_emu builds the CUDA sources into a CPU library to CHECK them; it is never a way to run
            raise EngineError(f"{_SO} is the SIMT-emulated test build of the engine; the product only runs on a CUDA "
                              "device (set B200NB_TEST_EMULATOR=1 only inside the test-suite)")
        for name, argt in SIGNATURES.items():
            f = getattr(l, name)
            f.argtypes = argt
            f.restype = _RESTYPE.get(name, C.c_int)
        _lib = l
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise EngineError(f"{what} failed: {lib().b200nb_last_error().decode()}")


def require_device() -> None:
    if lib().b200nb_device_count() < 1:
        raise EngineError("no CUDA device visible: the NB-GLM engine has no CPU fallback")
