"""Device-resident calls into the engine: torch tensors in, torch tensors out, nothing touches the host.

torch is plumbing here (allocation, streams); the work is the *_dev entry points of libb200nb.so.
Layout ("gene-major"): an n x m matrix is a torch tensor of shape (n, ld) whose first m columns are valid,
row-major, ld % 4 == 0 -- one gene per row, sample axis contiguous (include/b200nb.h).  Coefficient matrices
(beta, beta_var) are kept in R's column-major n x p form, i.e. a contiguous torch tensor of shape (p, n).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

F64 = torch.float64


def ld_for(m: int) -> int:
    return (m + 3) & ~3


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def to_gene_major(a, device="cuda"):
    """numpy (n, m) matrix (any order) -> device tensor (n, ld) in gene-major layout, dtype int32 or float64."""
    a = np.asarray(a)
    if np.issubdtype(a.dtype, np.integer):
        a = a.astype(np.int32, copy=False)
        dt = torch.int32
    else:
        a = a.astype(np.float64, copy=False)
        dt = F64
    n, m = a.shape
    out = torch.zeros((n, ld_for(m)), dtype=dt, device=device)
    out[:, :m] = torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return out


def colmajor_to_gene_major(src, n, m):
    """device column-major n x m buffer (flat tensor, R layout) -> gene-major (n, ld) via the engine's transpose."""
    L = _lib.lib()
    ld = ld_for(m)
    dst = torch.empty((n, ld), dtype=src.dtype, device=src.device)
    _lib.check(L.b200nb_to_gene_major_dev(_p(src), _p(dst), n, m, ld, src.element_size(), _stream()), "to_gene_major")
    return dst


def gene_major_to_colmajor(src, n, m):
    L = _lib.lib()
    dst = torch.empty(n * m, dtype=F64, device=src.device)
    _lib.check(L.b200nb_to_col_major_dev(_p(src), _p(dst), n, m, src.shape[1], _stream()), "to_col_major")
    return dst


def _ytype(y):
    if y.dtype == torch.int32:
        return 0
    if y.dtype == F64:
        return 1
    raise TypeError("y must be int32 or float64")


def _split_factors(sfd):
    """(size_factors, nf) for the entry points that take exactly one: sfd is the (m,) size-factor vector or the
    gene-major (n, ld) normalization-factor matrix."""
    return (None, sfd) if sfd.dim() == 2 else (sfd, None)


def fit_disp(y, x, mu_hat, log_alpha, log_alpha_prior_mean, log_alpha_prior_sigmasq, min_log_alpha, kappa_0, tol,
             maxit, usePrior, weights=None, weightThreshold=1e-2, useCR=True, m=None, out=None):
    """fitDisp on device tensors (src/DESeq2.cpp:164).  x: (m, p) numpy or tensor (column-major on device).
    Returns dict of device tensors with the reference's nine list member names."""
    L = _lib.lib()
    n, ld = y.shape
    xd = _x_dev(x, y.device)
    p, m_ = xd.shape
    m = m_ if m is None else m
    dev = y.device
    if out is None:
        out = {k: torch.empty(n, dtype=F64, device=dev) for k in
               ("log_alpha", "last_change", "initial_lp", "initial_dlp", "last_lp", "last_dlp", "last_d2lp")}
        out["iter"] = torch.empty(n, dtype=torch.int32, device=dev)
        out["iter_accept"] = torch.empty(n, dtype=torch.int32, device=dev)
    rc = L.b200nb_fit_disp_dev(_p(y), _ytype(y), _p(xd), _p(mu_hat), _p(log_alpha), _p(log_alpha_prior_mean),
                               float(log_alpha_prior_sigmasq), float(min_log_alpha), float(kappa_0), float(tol),
                               int(maxit), int(bool(usePrior)), _p(weights), int(weights is not None),
                               float(weightThreshold), int(bool(useCR)), n, m, p, ld,
                               _p(out["log_alpha"]), _p(out["iter"]), _p(out["iter_accept"]), _p(out["last_change"]),
                               _p(out["initial_lp"]), _p(out["initial_dlp"]), _p(out["last_lp"]), _p(out["last_dlp"]),
                               _p(out["last_d2lp"]), _stream())
    _lib.check(rc, "fit_disp_dev")
    return out


def fit_disp_grid(y, x, mu_hat, disp_grid, log_alpha_prior_mean, log_alpha_prior_sigmasq, usePrior, weights=None,
                  weightThreshold=1e-2, useCR=True):
    L = _lib.lib()
    n, ld = y.shape
    xd = _x_dev(x, y.device)
    p, m = xd.shape
    grid = disp_grid if isinstance(disp_grid, torch.Tensor) else torch.as_tensor(
        np.asarray(disp_grid, dtype=np.float64), device=y.device)
    la = torch.empty(n, dtype=F64, device=y.device)
    rc = L.b200nb_fit_disp_grid_dev(_p(y), _ytype(y), _p(xd), _p(mu_hat), _p(grid), grid.numel(),
                                    _p(log_alpha_prior_mean), float(log_alpha_prior_sigmasq), int(bool(usePrior)),
                                    _p(weights), int(weights is not None), float(weightThreshold), int(bool(useCR)),
                                    n, m, p, ld, _p(la), _stream())
    _lib.check(rc, "fit_disp_grid_dev")
    return {"log_alpha": la}


def fit_beta(y, x, nf, alpha_hat, contrast, beta_mat, lambda_, tol, maxit, useQR=True, minmu=0.5, weights=None,
             want_hat=True, want_mu=True, out=None, out_mu=None):
    """fitBeta on device tensors (src/DESeq2.cpp:283).  nf: (m,) size-factor vector or gene-major (n, ld) matrix.
    beta_mat: (p, n) contiguous (= column-major n x p).  out_mu: an (n, ld) buffer for the fitted mean (when out is
    not given)."""
    L = _lib.lib()
    n, ld = y.shape
    xd = _x_dev(x, y.device)
    p, m = xd.shape
    dev = y.device
    nf_is_vector = int(nf.dim() == 1)
    # pass device tensors to keep the call asynchronous (a numpy argument costs a synchronous pageable H2D copy)
    if not isinstance(contrast, torch.Tensor):
        contrast = torch.as_tensor(np.asarray(contrast, dtype=np.float64), device=dev)
    lam = lambda_ if isinstance(lambda_, torch.Tensor) else torch.as_tensor(np.asarray(lambda_, dtype=np.float64), device=dev)
    if out is None:
        out = {"beta_mat": torch.empty((p, n), dtype=F64, device=dev),
               "beta_var_mat": torch.empty((p, n), dtype=F64, device=dev),
               "iter": torch.empty(n, dtype=F64, device=dev),
               "contrast_num": torch.empty(n, dtype=F64, device=dev),
               "contrast_denom": torch.empty(n, dtype=F64, device=dev),
               "deviance": torch.empty(n, dtype=F64, device=dev),
               "hat_diagonals": torch.empty((n, ld), dtype=F64, device=dev) if want_hat else None,
               "mu": out_mu if out_mu is not None else (torch.empty((n, ld), dtype=F64, device=dev) if want_mu
                                                        else None)}
    rc = L.b200nb_fit_beta_dev(_p(y), _ytype(y), _p(xd), _p(nf), nf_is_vector, _p(alpha_hat), _p(contrast),
                               _p(beta_mat), _p(lam), _p(weights), int(weights is not None), float(tol), int(maxit),
                               int(bool(useQR)), float(minmu), n, m, p, ld, _p(out["beta_mat"]),
                               _p(out["beta_var_mat"]), _p(out["iter"]), _p(out["hat_diagonals"]),
                               _p(out["contrast_num"]), _p(out["contrast_denom"]), _p(out["deviance"]), _p(out["mu"]),
                               _stream())
    _lib.check(rc, "fit_beta_dev")
    return out


def beta_optim(y, x, nf, alpha_hat, lambda_nat, beta_start, weights=None, maxit=200):
    """b200nb_beta_optim_dev: fitNbinomGLMsOptim (R/fitNbinomGLMs.R:340-407) on the (few) rows passed in.
    beta_start: (p, n) contiguous, natural-log scale.  Returns {"beta_mat": (p, n), "converged": (n,) int32, "iter"}."""
    L = _lib.lib()
    n, ld = y.shape
    xd = _x_dev(x, y.device)
    p, m = xd.shape
    lam = lambda_nat if isinstance(lambda_nat, torch.Tensor) else torch.as_tensor(
        np.asarray(lambda_nat, dtype=np.float64), device=y.device)
    out = {"beta_mat": torch.empty((p, n), dtype=F64, device=y.device),
           "converged": torch.zeros(n, dtype=torch.int32, device=y.device),
           "iter": torch.zeros(n, dtype=torch.int32, device=y.device)}
    rc = L.b200nb_beta_optim_dev(_p(y), _ytype(y), _p(xd), _p(nf), int(nf.dim() == 1), _p(alpha_hat), _p(lam),
                                 _p(beta_start), _p(weights), int(weights is not None), int(maxit), n, m, p, ld,
                                 _p(out["beta_mat"]), _p(out["converged"]), _p(out["iter"]), _stream())
    _lib.check(rc, "beta_optim_dev")
    return out


def nb_loglik(y, x, nf, alpha_hat, beta_mat, weights=None, want_mu=True, out_mu=None, minmu=0.0):
    """b200nb_nb_loglik_dev: the unclamped fitted mean nf * exp(x beta) and nbinomLogLike at it -- what R recomputes
    right after fitBeta (R/fitNbinomGLMs.R:180-182).  beta_mat: (p, n) contiguous, natural-log scale.
    Returns {"logLike": (n,), "mu": (n, ld) or None}."""
    L = _lib.lib()
    n, ld = y.shape
    xd = _x_dev(x, y.device)
    p, m = xd.shape
    ll = torch.empty(n, dtype=F64, device=y.device)
    mu = out_mu if out_mu is not None else (torch.empty((n, ld), dtype=F64, device=y.device) if want_mu else None)
    rc = L.b200nb_nb_loglik_dev(_p(y), _ytype(y), _p(xd), _p(nf), int(nf.dim() == 1), _p(alpha_hat), _p(beta_mat),
                                _p(weights), int(weights is not None), float(minmu), n, m, p, ld, _p(ll), _p(mu),
                                _stream())
    _lib.check(rc, "nb_loglik_dev")
    return {"logLike": ll, "mu": mu}


def x_to_device(x, device="cuda"):
    """design matrix (m, p) numpy -> device tensor of shape (p, m) contiguous == R's column-major m x p."""
    return torch.as_tensor(np.ascontiguousarray(np.asarray(x, dtype=np.float64).T), device=device)


def _x_dev(x, device):
    return x if isinstance(x, torch.Tensor) else x_to_device(x, device)
