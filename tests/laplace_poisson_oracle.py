"""TEST INFRASTRUCTURE ONLY. Laplace approximation for a latent Vecchia GP with a poisson likelihood (log link): the numpy/scipy
restatement of oracle/laplace.py (bernoulli_logit) with the likelihood pieces exchanged. Every solve, the SLQ and the trace
machinery are oracle/laplace.py's own functions; only what depends on the likelihood is stated here:
  LogLikPoisson (without the constant)   include/GPBoost/likelihoods.h:11121-11126, 11407-11415
  normalising constant -sum log(y_i!)    include/GPBoost/likelihoods.h:10750-10757, 10985-10996, added to every sum at :11290
  first derivative y - exp(loc)          include/GPBoost/likelihoods.h:12176-12182, 12481-12483
  information W = exp(loc)               include/GPBoost/likelihoods.h:12881-12886, 13315-13317
  dW/dloc = exp(loc)                     include/GPBoost/likelihoods.h:13822-13827, 14110-14115
Pinned against the reference library by tests/golden/make_laplace_poisson_golden.py -> tests/golden/laplace_poisson_golden.json
(tests/test_laplace_poisson_oracle_pinned.py)."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from oracle import laplace as ol


def log_norm_const(y):
    """-sum_i log(y_i!) with each term summed as LogNormalizingConstantPoissonOneSample does (log 2 + log 3 + ... + log y_i)."""
    yi = np.asarray(y).astype(np.int64)
    lf = np.concatenate([[0., 0.], np.cumsum(np.log(np.arange(2, max(int(yi.max()), 1) + 1, dtype=np.float64)))])
    return float(np.sum(-lf[yi]))


def loglik(y, loc, cst):
    """LogLikelihood: sum_i (y_i loc_i - exp(loc_i)), then + log_normalizing_constant_."""
    return float(np.sum(y * loc - np.exp(loc))) + cst


def negll(coords_ordered, nn, cid, var, range_trans, y, fixed_effects=None, method="cholesky", probes=None, **kw):
    """Laplace-approximated negative marginal log-likelihood; returns dict(negll, mode, newton_it, cg_it, slq_it, logdet)
    (the keys of oracle.laplace.negll)."""
    cfg = dict(ol.DEFAULTS); cfg.update(kw)
    cst = log_norm_const(y)
    n = y.shape[0]
    A, Dinv, bad = ol.factor_latent(coords_ordered, nn, cid, var, range_trans)
    assert bad == 0
    B = ol.build_B(np.asarray(nn), A)
    Bt = B.T.tocsr()
    F = np.zeros(n) if fixed_effects is None else fixed_effects
    mode = np.zeros(n)
    SigmaI = (Bt @ sp.diags(Dinv) @ B).tocsc() if method == "cholesky" else None
    quad = lambda v: float((B @ v) @ (Dinv * (B @ v)))
    mll = loglik(y, F + mode, cst) - 0.5 * quad(mode)
    upd = np.zeros(n)
    cg_total = 0
    for it in range(cfg["maxit_mode_newton"]):
        W = np.exp(F + mode)
        rhs = W * mode + (y - W)
        if method == "cholesky":
            upd = spl.splu((SigmaI + sp.diags(W)).tocsc()).solve(rhs)
        else:
            upd, k = ol.cg_vadu(B, Bt, Dinv, W, rhs, upd, cfg["cg_max_num_it"], cfg["cg_delta_conv"], it == 0)
            cg_total += k
        direction = upd - mode
        gdd = float(direction @ (Bt @ (Dinv * (B @ direction)) + W * direction))
        lr = 1.
        for ih in range(cfg["max_lr_shrink"]):
            mode_new = upd if ih == 0 else (1 - lr) * mode + lr * upd
            mll_new = loglik(y, F + mode_new, cst) - 0.5 * quad(mode_new)
            if mll_new < mll + cfg["c_armijo"] * lr * gdd or not np.isfinite(mll_new):
                lr *= 0.5
            else:
                break
        mode = mode_new
        if it == 0:
            stop = abs(mll_new - mll) < cfg["delta_conv_mode_finding"] * abs(mll)
        else:
            stop = (mll_new - mll) < cfg["delta_conv_mode_finding"] * abs(mll)
        mll = mll_new
        if stop:
            break
    W = np.exp(F + mode)
    out = dict(mode=mode, newton_it=it, cg_it=cg_total, mll_mode=mll)
    if method == "cholesky":
        lu = spl.splu((SigmaI + sp.diags(W)).tocsc())
        logdet_A = float(np.sum(np.log(np.abs(lu.U.diagonal()))) + np.sum(np.log(np.abs(lu.L.diagonal()))))
        ld = logdet_A - float(np.sum(np.log(Dinv)))
        out["slq_it"] = 0
    else:
        t = cfg["num_rand_vec_trace"]
        if probes is None:
            probes = ol.gen_rand_normal(cfg["seed_rand_vec_trace"], 0, n, t)
        dw = Dinv + W
        Zp = Bt @ (np.sqrt(dw)[:, None] * probes)
        Td, Ts, its, AinvZ = ol.cg_tridiag_vadu(B, Bt, Dinv, W, Zp, min(cfg["cg_max_num_it_tridiag"], n), cfg["cg_delta_conv"])
        out["_Zp"], out["_AinvZ"] = Zp, AinvZ
        ld = ol.logdet_tridiag(Td, Ts, n) - float(np.sum(np.log(Dinv))) + float(np.sum(np.log(dw)))
        out["slq_it"] = its
    out["logdet"] = ld
    out["negll"] = -(mll - 0.5 * ld)
    out["_state"] = dict(A=A, Dinv=Dinv, B=B, Bt=Bt, W=W, F=F, cfg=cfg)
    return out


def grad_negll(coords_ordered, nn, cid, var, range_trans, y, fixed_effects=None, method="cholesky", probes=None, **kw):
    """Gradient w.r.t. (log variance, log range) at the mode, as oracle.laplace.grad_negll (same branches, same scale of the
    reference's optimiser in "grad", the derivative of this module's likelihood in "grad_consistent"), with dW = exp(loc)."""
    res = negll(coords_ordered, nn, cid, var, range_trans, y, fixed_effects=fixed_effects, method=method, probes=probes, **kw)
    st = res["_state"]
    B, Bt, Dinv, W, cfg = st["B"], st["Bt"], st["Dinv"], st["W"], st["cfg"]
    n = y.shape[0]
    mode = res["mode"]
    _, Dinv2, Ag, Dg, bad = ol.factor_latent_grad(coords_ordered, nn, cid, var, range_trans)
    assert bad == 0 and np.allclose(Dinv2, Dinv, rtol=0, atol=0)
    nn = np.asarray(nn)
    m = nn.shape[1]
    rows = np.repeat(np.arange(n), m)
    mask = nn.ravel() >= 0
    Bg = sp.csr_matrix((-Ag.ravel()[mask], (rows[mask], nn.ravel()[mask])), shape=(n, n))  # B_grad (zero diagonal)
    Dm = sp.diags(Dinv)
    SigmaI = (Bt @ Dm @ B).tocsr()
    X1 = (Bg.T @ Dm @ B)
    SigmaI_deriv = [(-SigmaI).tocsr(), (X1 + X1.T - Bt @ sp.diags(Dinv * Dg * Dinv) @ B).tocsr()]
    dW = np.exp(st["F"] + mode)  # CalcFirstDerivInformationLocPar, poisson
    grad = np.zeros(2)
    if method == "cholesky":
        Ainv = np.linalg.inv((SigmaI + sp.diags(W)).toarray())
        d_mll_d_mode = 0.5 * np.diag(Ainv) * dW
        Ainv_dmll = Ainv @ d_mll_d_mode
        for j in range(2):
            Sd = SigmaI_deriv[j]
            Sd_mode = Sd @ mode
            explicit = 0.5 * (mode @ Sd_mode + float(Sd.multiply(Ainv).sum()))
            explicit += 0.5 * n if j == 0 else 0.5 * float(np.sum(Dinv * Dg))
            grad[j] = explicit - Ainv_dmll @ Sd_mode
    else:
        Zp, AinvZ = res["_Zp"], res["_AinvZ"]
        dw = Dinv + W
        PI_Z = ol._vadu_solve(B, Bt, dw, Zp)
        ZA = AinvZ * dW[:, None] * PI_Z
        trA = ZA.mean(1)
        Dw_inv = 1. / dw
        trD = Dw_inv * dW
        BPZ = B @ PI_Z
        ZP = BPZ * dW[:, None] * BPZ
        trP = ZP.mean(1)
        cA = ZA - trA[:, None]; cP = ZP - trP[:, None]
        c_var = (cP * cP).mean(1)
        with np.errstate(divide="ignore", invalid="ignore"):
            c_opt = np.where(c_var == 0, 1., (cA * cP).mean(1) / c_var)
        d_mll_d_mode = 0.5 * (trA + c_opt * trD - c_opt * trP)
        Ainv_dmll, _ = ol.cg_vadu(B, Bt, Dinv, W, d_mll_d_mode, np.zeros(n), cfg["cg_max_num_it"], cfg["cg_delta_conv"], True)
        for j in range(2):
            Sd = SigmaI_deriv[j]
            zA = (AinvZ * (Sd @ PI_Z)).sum(0)
            tr1 = float(zA.mean())
            d = tr1 + (n if j == 0 else float(np.sum(Dinv * Dg)))
            if j == 0:
                trDd = -float(np.sum(Dw_inv * Dinv))
                zP = (PI_Z * (Sd @ PI_Z)).sum(0)
            else:
                trDd = -float(np.sum(Dw_inv * Dinv * Dg * Dinv))
                BtWBg = (Bt @ sp.diags(W) @ Bg)
                Pd = (Sd + BtWBg.T + BtWBg).tocsr()
                zP = (PI_Z * (Pd @ PI_Z)).sum(0)
            trPd = float(zP.mean())
            c = ol._optimal_c(zA, zP, tr1, trPd)
            d += c * trDd - c * trPd
            Sd_mode = Sd @ mode
            grad[j] = 0.5 * (mode @ Sd_mode + d) - Ainv_dmll @ Sd_mode
    # scale of the reference's optimiser (log of the original range), as in oracle.laplace.grad_negll
    res["grad_trans"] = grad.copy()
    res["grad_consistent"] = grad * np.array([1., -2. if cid == 3 else -1.])
    grad[1] *= -0.5 if cid == 3 else -1.
    res["grad"] = grad
    return res
