"""torch-tensor front end of the device layer (pdsb_dev_*).  torch is plumbing here: it owns device memory and
streams (and torch.distributed carries the one collective of the multi-GPU path); all arithmetic is in the library.

Layout convention: a design matrix is a torch tensor of shape (p, ld) — p columns of ld >= n rows, row-major in
torch == column-major [ld x p] for the library.  Targets likewise (t, ld).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from ._lib import (DT_BOOL, DT_F32, DT_F64, DT_I8, DT_I16, DT_I32, DT_I64, DT_U8, DT_U16, DT_U32, DT_U64,
                   METHOD_CD, METHOD_INV, METHOD_LSTSQ, METHOD_NNLS, METHOD_RCOND, SOLVER_CHOLESKEY, SOLVER_QR,
                   SOLVER_SVD, Chunk, Column, SolveOpts, check, lib)


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _sfx(t: torch.Tensor) -> str:
    if t.dtype == torch.float32:
        return "f32"
    if t.dtype == torch.float64:
        return "f64"
    raise TypeError(f"unsupported dtype {t.dtype}")


def _ld(t: torch.Tensor) -> int:
    assert t.dim() == 2 and t.stride(1) == 1, "matrix must be (columns, rows) with contiguous rows"
    return t.stride(0) if t.shape[0] > 1 else t.shape[1]


def moments(X: torch.Tensor, Y: torch.Tensor, n: Optional[int] = None, w: Optional[torch.Tensor] = None,
            mask: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """M = [X|Y|1]^T diag(w) [X|Y|1] as a (q1, q1) float64 tensor, q1 = p + t + 1."""
    p, t = X.shape[0], Y.shape[0]
    n = X.shape[1] if n is None else n
    q1 = p + t + 1
    M = out if out is not None else torch.empty((q1, q1), dtype=torch.float64, device=X.device)
    fn = getattr(lib(), f"pdsb_dev_moments_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(Y), _ld(Y), _ptr(w), _ptr(mask), n, p, t, _ptr(M), _stream()))
    return M


def solve(M: torch.Tensor, p: int, t: int = 1, add_bias: bool = False, method: int = METHOD_LSTSQ,
          solver: int = SOLVER_QR, l1_reg: float = 0.0, l2_reg: float = 0.0, tol: float = 0.0,
          singular_x_tol: float = 0.0, positive: bool = False, max_iter: int = 200, want_aux: bool = False,
          beta: Optional[torch.Tensor] = None, status: Optional[torch.Tensor] = None):
    q = p + int(add_bias)
    beta = beta if beta is not None else torch.empty((t, q), dtype=torch.float64, device=M.device)
    status = status if status is not None else torch.zeros(4, dtype=torch.int32, device=M.device)
    aux = torch.zeros(q * q + q, dtype=torch.float64, device=M.device) if want_aux else None
    o = SolveOpts(p=p, t=t, add_bias=int(add_bias), method=method, solver=solver, positive=int(positive),
                  max_iter=max_iter, f32_gate=0, l1_reg=l1_reg, l2_reg=l2_reg, tol=tol, singular_x_tol=singular_x_tol)
    check(lib().pdsb_dev_solve(_ptr(M), C.byref(o), _ptr(beta), _ptr(status), _ptr(aux), _stream()))
    return (beta, status, aux) if want_aux else (beta, status)


def predict(X: torch.Tensor, Y: torch.Tensor, beta: torch.Tensor, status: Optional[torch.Tensor], add_bias: bool,
            n: Optional[int] = None, mask: Optional[torch.Tensor] = None, w: Optional[torch.Tensor] = None,
            pred: Optional[torch.Tensor] = None, resid: Optional[torch.Tensor] = None,
            valid: Optional[torch.Tensor] = None, ssr: Optional[torch.Tensor] = None):
    p, t = X.shape[0], Y.shape[0]
    n = X.shape[1] if n is None else n
    ld = _ld(X)
    pred = pred if pred is not None else torch.empty((t, ld), dtype=X.dtype, device=X.device)
    resid = resid if resid is not None else torch.empty((t, ld), dtype=X.dtype, device=X.device)
    fn = getattr(lib(), f"pdsb_dev_predict_{_sfx(X)}")
    check(fn(_ptr(X), ld, _ptr(Y), _ld(Y), _ptr(w), _ptr(mask), n, p, t, int(add_bias), _ptr(beta), _ptr(status),
             _ptr(pred), _ptr(resid), _ld(pred), _ptr(valid), _ptr(ssr), _stream()))
    return pred, resid


def grouped_lin_reg(X: torch.Tensor, y: torch.Tensor, offsets: torch.Tensor, add_bias: bool = False,
                    l2_reg: float = 0.0, singular_x_tol: float = 0.0, solver: int = SOLVER_QR,
                    method: int = METHOD_LSTSQ, l1_reg: float = 0.0, positive: bool = False, tol: float = 0.0,
                    max_iter: int = 200):
    """Every group's lin_reg fit: (beta (n_groups, p + bias) float64, status (n_groups,) int32).  method: METHOD_LSTSQ
    (solver, l2_reg, singular_x_tol), or METHOD_CD (l1_reg, l2_reg, positive) / METHOD_NNLS, which iterate up to
    max_iter sweeps and stop early once a sweep moves no coefficient by tol or more (CD) / the KKT conditions hold to
    tol (NNLS)."""
    p = X.shape[0]
    n = X.shape[1]
    ng = offsets.numel() - 1
    q = p + int(add_bias)
    beta = torch.empty((ng, q), dtype=torch.float64, device=X.device)
    status = torch.empty(ng, dtype=torch.int32, device=X.device)
    o = SolveOpts(p=p, t=1, add_bias=int(add_bias), method=method, solver=solver, positive=int(positive),
                  max_iter=max_iter, l1_reg=l1_reg, l2_reg=l2_reg, tol=tol, singular_x_tol=singular_x_tol)
    fn = getattr(lib(), f"pdsb_dev_grouped_lin_reg_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(y), _ptr(offsets), ng, n, p, C.byref(o), _ptr(beta), _ptr(status), _stream()))
    return beta, status


def grouped_wls_lin_reg(X: torch.Tensor, y: torch.Tensor, w: torch.Tensor, offsets: torch.Tensor,
                        add_bias: bool = False, l2_reg: float = 0.0, singular_x_tol: float = 0.0,
                        solver: int = SOLVER_QR):
    """Every group's weighted least squares: grouped_lin_reg's fit (METHOD_LSTSQ) on moments weighted by w (length n,
    X's dtype).  A row with a NaN / inf in x, y or w is dropped; a group with fewer kept rows than coefficients gets a
    nonzero status and NaN beta.  w = 1 gives grouped_lin_reg's result bit for bit.  The single weighted fit uses
    l2_reg = 0 and singular_x_tol = 0.  Returns (beta (n_groups, p + bias) float64, status (n_groups,) int32)."""
    p = X.shape[0]
    n = X.shape[1]
    ng = offsets.numel() - 1
    q = p + int(add_bias)
    beta = torch.empty((ng, q), dtype=torch.float64, device=X.device)
    status = torch.empty(ng, dtype=torch.int32, device=X.device)
    o = SolveOpts(p=p, t=1, add_bias=int(add_bias), method=METHOD_LSTSQ, solver=solver, l2_reg=l2_reg,
                  singular_x_tol=singular_x_tol)
    fn = getattr(lib(), f"pdsb_dev_grouped_wls_lin_reg_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(y), _ptr(w), _ptr(offsets), ng, n, p, C.byref(o), _ptr(beta), _ptr(status),
             _stream()))
    return beta, status


def grouped_lin_reg_multi(Z: torch.Tensor, offsets: torch.Tensor, n_targets: int, add_bias: bool = False,
                          l2_reg: float = 0.0, singular_x_tol: float = 0.0, solver: int = SOLVER_QR):
    """Every group's multi-target fit from one read of Z (t + p, ld) = [y_0 .. y_{t-1} | x_0 .. x_{p-1}], t =
    ``n_targets``: target c of group g is grouped_lin_reg's fit of y_c on X over rows [offsets[g], offsets[g+1]).  A row
    with a NaN / inf anywhere is dropped for every target.  Returns (beta (n_groups, t, p + bias) float64, status
    (n_groups,) int32; a nonzero status nulls every target of its group)."""
    t = n_targets
    p = Z.shape[0] - t
    n = Z.shape[1]
    ng = offsets.numel() - 1
    q = p + int(add_bias)
    beta = torch.empty((ng, t, q), dtype=torch.float64, device=Z.device)
    status = torch.empty(ng, dtype=torch.int32, device=Z.device)
    o = SolveOpts(p=p, t=t, add_bias=int(add_bias), method=METHOD_LSTSQ, solver=solver, l2_reg=l2_reg,
                  singular_x_tol=singular_x_tol)
    fn = getattr(lib(), f"pdsb_dev_grouped_lin_reg_multi_{_sfx(Z)}")
    check(fn(_ptr(Z), _ld(Z), t, p, _ptr(offsets), ng, n, C.byref(o), _ptr(beta), _ptr(status), _stream()))
    return beta, status


def grouped_ar_coeffs(x: torch.Tensor, offsets: torch.Tensor, lag: int, add_bias: bool = True,
                      mask: Optional[torch.Tensor] = None, l2_reg: float = 0.0,
                      singular_x_tol: Optional[float] = None, solver: int = SOLVER_QR):
    """Every group's autoregression of order ``lag`` from the one column x (group g = x[offsets[g]:offsets[g+1]]): the
    fit of grouped_lin_reg on the group's lagged design (target rows t = lag.., features x_{t-1} .. x_{t-lag}), formed on
    the device.  mask (optional, 0 / 1 per row): 0 drops row t as a target; x_t stays a lag of the rows after it.
    singular_x_tol defaults to lin_reg's for x's dtype.  Returns (beta [n_groups, lag + bias] float64, status)."""
    ng = offsets.numel() - 1
    q = lag + int(add_bias)
    if singular_x_tol is None:
        singular_x_tol = 1e-6 if x.dtype == torch.float32 else 1e-12
    beta = torch.empty((ng, q), dtype=torch.float64, device=x.device)
    status = torch.empty(ng, dtype=torch.int32, device=x.device)
    o = SolveOpts(p=lag, t=1, add_bias=int(add_bias), method=METHOD_LSTSQ, solver=solver, l2_reg=l2_reg,
                  singular_x_tol=singular_x_tol)
    fn = getattr(lib(), f"pdsb_dev_grouped_ar_lin_reg_{_sfx(x)}")
    check(fn(_ptr(x), _ptr(mask), _ptr(offsets), ng, x.numel(), lag, C.byref(o), _ptr(beta), _ptr(status), _stream()))
    return beta, status


def grouped_lin_reg_rcond(X: torch.Tensor, y: torch.Tensor, offsets: torch.Tensor, add_bias: bool = False,
                          rcond: float = 0.0, l2_reg: float = 0.0):
    """Every group's lin_reg_w_rcond fit (K19): (beta (n_groups, p + bias) float64, singular values (n_groups, p + bias)
    float64 in descending order, status (n_groups,) int32).  Group g is rows [offsets[g], offsets[g+1]) of X (p, ld) / y,
    null rows as NaN; each group's tolerance is max(|rcond|, eps * max(its rows, p + bias)) in X's dtype.  status 1
    (gated): fewer kept rows than coefficients, beta and the singular values are NaN."""
    p = X.shape[0]
    n = X.shape[1]
    ng = offsets.numel() - 1
    q = p + int(add_bias)
    beta = torch.empty((ng, q), dtype=torch.float64, device=X.device)
    sv = torch.empty((ng, q), dtype=torch.float64, device=X.device)
    status = torch.empty(ng, dtype=torch.int32, device=X.device)
    o = SolveOpts(p=p, t=1, add_bias=int(add_bias), method=METHOD_RCOND, l2_reg=l2_reg, tol=abs(rcond))
    fn = getattr(lib(), f"pdsb_dev_grouped_lin_reg_rcond_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(y), _ptr(offsets), ng, n, p, C.byref(o), _ptr(beta), _ptr(sv), _ptr(status),
             _stream()))
    return beta, sv, status


def grouped_predict(X: torch.Tensor, y: torch.Tensor, offsets: torch.Tensor, beta: torch.Tensor, status: torch.Tensor,
                    add_bias: bool, mask: Optional[torch.Tensor] = None, n: Optional[int] = None,
                    pred: Optional[torch.Tensor] = None, resid: Optional[torch.Tensor] = None,
                    valid: Optional[torch.Tensor] = None):
    """pred / resid / valid of every row of the groups [offsets[g], offsets[g+1]) with the beta / status of
    grouped_lin_reg: (pred, resid, valid), each of length n."""
    p = X.shape[0]
    n = X.shape[1] if n is None else n
    ng = offsets.numel() - 1
    pred = pred if pred is not None else torch.empty(n, dtype=X.dtype, device=X.device)
    resid = resid if resid is not None else torch.empty(n, dtype=X.dtype, device=X.device)
    valid = valid if valid is not None else torch.empty(n, dtype=torch.uint8, device=X.device)
    fn = getattr(lib(), f"pdsb_dev_grouped_predict_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(y), _ptr(offsets), ng, n, p, int(add_bias), _ptr(beta), _ptr(status), _ptr(mask),
             _ptr(pred), _ptr(resid), _ptr(valid), _stream()))
    return pred, resid, valid


def grouped_logistic(X: torch.Tensor, y: torch.Tensor, offsets: torch.Tensor, add_bias: bool = True,
                     l1_reg: float = 0.0, l2_reg: float = 0.0, tol: float = 1e-5, max_iter: int = 200,
                     mask: Optional[torch.Tensor] = None, n: Optional[int] = None):
    """Every group's logistic_reg fit, float64: (beta (n_groups, p + bias), status (n_groups,) int32, iterations run).
    status: LOGISTIC_CONVERGED / _MAX_ITER / _FAILED / _EMPTY (_lib); beta is NaN for a failed or empty group."""
    p = X.shape[0]
    n = X.shape[1] if n is None else n
    ng = offsets.numel() - 1
    beta = torch.empty((ng, p + int(add_bias)), dtype=torch.float64, device=X.device)
    status = torch.empty(ng, dtype=torch.int32, device=X.device)
    n_iter = C.c_int64(0)
    check(lib().pdsb_dev_grouped_logistic_f64(_ptr(X), _ld(X), _ptr(y), _ptr(mask), _ptr(offsets), ng, n, p,
                                              int(add_bias), float(l1_reg), float(l2_reg), float(tol), int(max_iter),
                                              _ptr(beta), _ptr(status), C.byref(n_iter), _stream()))
    return beta, status, int(n_iter.value)


def grouped_glm(X: torch.Tensor, y: torch.Tensor, offsets: torch.Tensor, family: int, add_bias: bool = False,
                tol: float = 1e-8, max_iter: int = 100, mask: Optional[torch.Tensor] = None, n: Optional[int] = None):
    """Every group's GLM.fit, float64: (beta (n_groups, p + bias), status (n_groups,) int32, n_iter (n_groups,) int64).
    family: GLM_GAUSSIAN / _POISSON / _BINOMIAL / _GAMMA; status: GLM_CONVERGED / _MAX_ITER / _FAILED / _EMPTY (_lib);
    beta is NaN for a failed or empty group."""
    p = X.shape[0]
    n = X.shape[1] if n is None else n
    ng = offsets.numel() - 1
    beta = torch.empty((ng, p + int(add_bias)), dtype=torch.float64, device=X.device)
    status = torch.empty(ng, dtype=torch.int32, device=X.device)
    n_iter = torch.empty(ng, dtype=torch.int64, device=X.device)
    check(lib().pdsb_dev_grouped_glm_f64(_ptr(X), _ld(X), _ptr(y), _ptr(mask), _ptr(offsets), ng, n, p, int(add_bias),
                                         int(family), float(tol), int(max_iter), _ptr(beta), _ptr(status), _ptr(n_iter),
                                         _stream()))
    return beta, status, n_iter


def grouped_report(X: torch.Tensor, y: torch.Tensor, offsets: torch.Tensor, add_bias: bool = False, se_type: int = 0,
                   ymask: Optional[torch.Tensor] = None, n: Optional[int] = None):
    """Every group's lin_reg_report block: (out (n_groups, 8, p + bias) float64, status (n_groups,) int32).  Group g is
    rows [offsets[g], offsets[g+1]) of X (p, ld) / y, null rows as NaN; ymask: the y validity (0 / 1) for var(y); se_type 0
    se, 1..4 hc0..hc3.  status 1 (gated): fewer kept rows than coefficients, the block is NaN."""
    p = X.shape[0]
    n = X.shape[1] if n is None else n
    ng = offsets.numel() - 1
    out = torch.empty((ng, 8, p + int(add_bias)), dtype=torch.float64, device=X.device)
    status = torch.empty(ng, dtype=torch.int32, device=X.device)
    fn = getattr(lib(), f"pdsb_dev_grouped_report_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(y), _ptr(ymask), _ptr(offsets), ng, n, p, int(add_bias), int(se_type), _ptr(out),
             _ptr(status), _stream()))
    return out, status


def grouped_pca(X: torch.Tensor, offsets: torch.Tensor, center: bool = True, mask: Optional[torch.Tensor] = None,
                n: Optional[int] = None):
    """Every group's PCA (K18): (mean (n_groups, p) float64 or None without centring, sigma (n_groups, p) float64,
    V (n_groups, p, p) float64 with V[g][:, r] = weight vector r, status (n_groups, 2) int32: PDSB_PCA_OK (0) or
    _NONFINITE (1), dim).  Group g is rows [offsets[g], offsets[g+1]) of X (p, ld); mask: per-row 0 / 1, masked rows leave
    the Gram and their NaN values are nulls for the means."""
    p = X.shape[0]
    n = X.shape[1] if n is None else n
    ng = offsets.numel() - 1
    dev = X.device
    mean = torch.empty((ng, p), dtype=torch.float64, device=dev) if center else None
    sigma = torch.empty((ng, p), dtype=torch.float64, device=dev)
    Vt = torch.empty((ng, p, p), dtype=torch.float64, device=dev)      # [g][r][i] = column r of V_g
    status = torch.empty((ng, 2), dtype=torch.int32, device=dev)
    fn = getattr(lib(), f"pdsb_dev_grouped_pca_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(mask), _ptr(offsets), ng, n, p, int(center), _ptr(mean), _ptr(sigma), _ptr(Vt),
             _ptr(status), _stream()))
    return mean, sigma, Vt.transpose(1, 2), status


def grouped_project(X: torch.Tensor, offsets: torch.Tensor, V: torch.Tensor, k: int,
                    mean: Optional[torch.Tensor] = None, n: Optional[int] = None) -> torch.Tensor:
    """(x_r - mean_g) V_g[:, :k] for every row of every group: (k, n) float64, NaN rows for a group with fewer than k
    rows.  V as grouped_pca returns it (n_groups, p, p); mean None: no centring."""
    p = X.shape[0]
    n = X.shape[1] if n is None else n
    ng = offsets.numel() - 1
    Vt = V.transpose(1, 2).contiguous()
    out = torch.empty((k, n), dtype=torch.float64, device=X.device)
    fn = getattr(lib(), f"pdsb_dev_grouped_project_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(offsets), ng, n, p, _ptr(mean), _ptr(Vt), int(k), _ptr(out), n, _stream()))
    return out


def online_lin_reg(X: torch.Tensor, y: torch.Tensor, window: int, min_rows: int, add_bias: bool = False,
                   l2_reg: float = 0.0, skip: bool = False, n: Optional[int] = None,
                   coeffs: Optional[torch.Tensor] = None, pred: Optional[torch.Tensor] = None,
                   valid: Optional[torch.Tensor] = None):
    """window > 0: rolling_lin_reg; window == 0: recursive_lin_reg starting after `min_rows` rows."""
    p = X.shape[0]
    n = X.shape[1] if n is None else n
    q = p + int(add_bias)
    coeffs = coeffs if coeffs is not None else torch.empty((n, q), dtype=X.dtype, device=X.device)
    pred = pred if pred is not None else torch.empty(n, dtype=X.dtype, device=X.device)
    valid = valid if valid is not None else torch.empty(n, dtype=torch.uint8, device=X.device)
    fn = getattr(lib(), f"pdsb_dev_online_lin_reg_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(y), n, p, int(add_bias), window, min_rows, int(skip), float(l2_reg), _ptr(coeffs),
             _ptr(pred), _ptr(valid), _stream()))
    return coeffs, pred, valid


def grouped_recursive_lin_reg(X: torch.Tensor, y: torch.Tensor, offsets: torch.Tensor, min_rows: int,
                              add_bias: bool = False, l2_reg: float = 0.0, skip: Optional[torch.Tensor] = None,
                              n: Optional[int] = None):
    """recursive_lin_reg(...).over(key): group g is rows [offsets[g], offsets[g+1]) (int64 on the device); per group,
    bit for bit ``online_lin_reg(window=0)`` on its rows, with ``skip[g]`` (uint8 per group, None: no group skips)."""
    p = X.shape[0]
    n = X.shape[1] if n is None else n
    q = p + int(add_bias)
    coeffs = torch.empty((n, q), dtype=X.dtype, device=X.device)
    pred = torch.empty(n, dtype=X.dtype, device=X.device)
    valid = torch.empty(n, dtype=torch.uint8, device=X.device)
    fn = getattr(lib(), f"pdsb_dev_grouped_recursive_lin_reg_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(y), n, p, int(add_bias), min_rows, float(l2_reg), _ptr(offsets), offsets.numel() - 1,
             _ptr(skip), _ptr(coeffs), _ptr(pred), _ptr(valid), _stream()))
    return coeffs, pred, valid


def grouped_rolling_lin_reg(X: torch.Tensor, y: torch.Tensor, offsets: torch.Tensor, window: int, min_rows: int,
                            add_bias: bool = False, l2_reg: float = 0.0, skip: Optional[torch.Tensor] = None,
                            n: Optional[int] = None):
    """rolling_lin_reg over groups: group g is rows [offsets[g], offsets[g+1]) (int64 on the device); per group, bit for
    bit ``online_lin_reg(window, min_rows)`` on its rows, with ``skip[g]`` (uint8 per group, None: no group skips)."""
    p = X.shape[0]
    n = X.shape[1] if n is None else n
    q = p + int(add_bias)
    coeffs = torch.empty((n, q), dtype=X.dtype, device=X.device)
    pred = torch.empty(n, dtype=X.dtype, device=X.device)
    valid = torch.empty(n, dtype=torch.uint8, device=X.device)
    fn = getattr(lib(), f"pdsb_dev_grouped_rolling_lin_reg_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(y), n, p, int(add_bias), int(window), int(min_rows), float(l2_reg), _ptr(offsets),
             offsets.numel() - 1, _ptr(skip), _ptr(coeffs), _ptr(pred), _ptr(valid), _stream()))
    return coeffs, pred, valid


def recursive_shard(X: torch.Tensor, y: torch.Tensor, min_rows: int, m0: Optional[torch.Tensor], row0: int,
                    add_bias: bool = False, l2_reg: float = 0.0, skip: bool = False):
    """recursive_lin_reg on the row shard that starts at global row `row0`; `m0` = float64 (p+2)^2 moments
    ([X | y | 1]) of all preceding rows (None for the first shard)."""
    p, n = X.shape
    q = p + int(add_bias)
    coeffs = torch.empty((n, q), dtype=X.dtype, device=X.device)
    pred = torch.empty(n, dtype=X.dtype, device=X.device)
    valid = torch.empty(n, dtype=torch.uint8, device=X.device)
    if m0 is not None:
        assert m0.dtype == torch.float64 and m0.is_contiguous() and m0.numel() == (p + 2) ** 2
    fn = getattr(lib(), f"pdsb_dev_recursive_shard_{_sfx(X)}")
    check(fn(_ptr(X), _ld(X), _ptr(y), n, p, int(add_bias), min_rows, int(skip), float(l2_reg),
             _ptr(m0) if m0 is not None else None, row0, _ptr(coeffs), _ptr(pred), _ptr(valid), _stream()))
    return coeffs, pred, valid


FRAME_ROWS = 128


def frame_elems(n: int, ncols: int) -> int:
    return int(lib().pdsb_frame_elems(n, ncols))


def to_frame(Z: torch.Tensor, n: Optional[int] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Column-major (ncols, ld) float32 matrix -> row-blocked frame [block][column][128] (flat tensor)."""
    ncols = Z.shape[0]
    n = Z.shape[1] if n is None else n
    frame = out if out is not None else torch.empty(frame_elems(n, ncols), dtype=torch.float32, device=Z.device)
    check(lib().pdsb_dev_frame_from_colmajor_f32(_ptr(Z), _ld(Z), n, ncols, _ptr(frame), _stream()))
    return frame


def moments_frame(frame: torch.Tensor, n: int, ncols: int, xcol: int, p: int, ycol: int, t: int = 1,
                  mask: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    q1 = p + t + 1
    M = out if out is not None else torch.empty((q1, q1), dtype=torch.float64, device=frame.device)
    check(lib().pdsb_dev_moments_frame_f32(_ptr(frame), n, ncols, xcol, p, ycol, t, _ptr(mask), _ptr(M), _stream()))
    return M


def predict_frame(frame: torch.Tensor, n: int, ncols: int, xcol: int, p: int, ycol: int, t: int, beta: torch.Tensor,
                  status: Optional[torch.Tensor], add_bias: bool, pred: torch.Tensor, resid: torch.Tensor,
                  mask: Optional[torch.Tensor] = None, valid: Optional[torch.Tensor] = None,
                  ssr: Optional[torch.Tensor] = None):
    check(lib().pdsb_dev_predict_frame_f32(_ptr(frame), n, ncols, xcol, p, ycol, t, int(add_bias), _ptr(mask), _ptr(beta),
                                           _ptr(status), _ptr(pred), _ptr(resid), _ld(pred), _ptr(valid), _ptr(ssr),
                                           _stream()))
    return pred, resid


_ARROW_DTYPES = {"float": DT_F32, "double": DT_F64, "int8": DT_I8, "uint8": DT_U8, "int16": DT_I16, "uint16": DT_U16,
                 "int32": DT_I32, "uint32": DT_U32, "int64": DT_I64, "uint64": DT_U64, "bool": DT_BOOL}


def _column(a, null_count: Optional[int], pinned: bool, keep: list) -> Column:
    """pa.Array / pa.ChunkedArray -> pdsb_column over its buffers (pageable, or page-locked copies with pinned=True).
    Unlike the plugin import, a chunk's validity buffer is passed whenever it exists, also when the chunk has no null."""
    import pyarrow as pa

    chunks = a.chunks if isinstance(a, pa.ChunkedArray) else [a]
    if str(a.type) not in _ARROW_DTYPES:
        raise TypeError(f"unsupported Arrow type {a.type}")
    arr = (Chunk * max(len(chunks), 1))()
    for j, ch in enumerate(chunks):
        bufs = ch.buffers()
        ptr = []
        for b in bufs[:2]:
            if b is None:
                ptr.append(None)
            elif pinned:
                t = torch.frombuffer(memoryview(b), dtype=torch.uint8).pin_memory() if b.size else torch.empty(
                    1, dtype=torch.uint8).pin_memory()
                keep.append(t)
                ptr.append(t.data_ptr())
            else:
                ptr.append(b.address)
        arr[j] = Chunk(ptr[1], ptr[0], ch.offset, len(ch))
    keep.append(arr)
    nc = a.null_count if null_count is None else null_count
    return Column(b"", _ARROW_DTYPES[str(a.type)], len(chunks), C.cast(arr, C.POINTER(Chunk)), nc)


def build_frame(columns, n_targets: int = 1, null_policy: str = "skip", dtype: torch.dtype = torch.float64,
                multi: bool = False, online: bool = False, weights=None, null_counts=None, pinned: bool = False,
                device: Optional[torch.device] = None):
    """The fits' frame builder on Arrow host columns (targets first, then features): (n, Z (n_cols, ld), mask (ld,) or
    None when no row is dropped, w (ld,) or None).  null_counts: per column, None = the array's own count, -1 = let
    the library count from the bitmaps.  Rows n..ld of the outputs are not defined."""
    keep: list = []
    ncs = null_counts if null_counts is not None else [None] * len(columns)
    cols = (Column * max(len(columns), 1))(*[_column(c, nc, pinned, keep) for c, nc in zip(columns, ncs)])
    wcol = _column(weights, None, pinned, keep) if weights is not None else None
    lens = [len(c) for c in columns] + ([len(weights)] if weights is not None else [])
    cap = max(32, (max(lens, default=0) + 31) // 32 * 32)
    dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
    Z = torch.empty((max(len(columns), 1), cap), dtype=dtype, device=dev)
    mask = torch.empty(cap, dtype=dtype, device=dev)
    w = torch.empty(cap, dtype=dtype, device=dev) if weights is not None else None
    n, ld, has_mask = C.c_int64(0), C.c_int64(0), C.c_int(0)
    fn = getattr(lib(), f"pdsb_dev_build_frame_{_sfx(Z)}")
    check(fn(cols, len(columns), n_targets, C.byref(wcol) if wcol is not None else None, null_policy.encode(),
             int(multi), int(online), cap, C.byref(n), C.byref(ld), _ptr(Z), _ptr(mask), C.byref(has_mask), _ptr(w),
             _stream()))
    del keep
    return int(n.value), Z[:len(columns), :ld.value], (mask[:ld.value] if has_mask.value else None), \
        (w[:ld.value] if w is not None else None)


def launch_count() -> int:
    return int(lib().pdsb_kernel_launch_count())
