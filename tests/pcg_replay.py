"""Float64 replays of the two solves of the reduced camera system (RCS: the 9 nc x 9 nc camera system left after the landmarks
are eliminated), iterate by iterate, on whatever operator, right-hand side and block-Jacobi inverse they are given.

pcg_replay follows the reference's ConjugateGradientsSolver::solve (cg/conjugate_gradient.hpp:113-298) line for line, driven
as LinearizorBase drives it (linearizor_base.cpp:81-103): x_0 = 0, r_tolerance = -1 (the residual test never fires), the
residual recomputed as b - H x every `period`-th iteration, the zeta rule of Nash & Sofer with its min_num_iterations gate,
and max_num_iterations.  It solves H x = b; the increment the solvers return is inc = -x.  Termination types are those of
rba_cg_summary: 0 NO_CONVERGENCE, 1 SUCCESS, 2 FAILURE.

power_replay follows LinearizationPowerSC::solve (sc/linearization_power_sc.hpp:127-158):
    accum = Hpp_d^-1 (-b);  tmp = accum;  for i = 1..order: tmp = Hpp_d^-1 (E0 tmp); accum += tmp;
    stop with SUCCESS when q_tolerance > 0 and i |tmp| / |accum| < q_tolerance.
accum is already the increment.  The solver exposes no E0 accessor, but it does not need one: for the Power-SC handle
right_multiply applies the RCS operator S = Hpp_d - E0 (Hpp_d = sum Jp^T Jp + lambda I, the damped camera blocks) and
get_preconditioner returns the block-diagonal Hpp_d^-1.  Hence
    Hpp_d^-1 E0 t = Hpp_d^-1 (Hpp_d t - S t) = t - Hpp_d^-1 (S t),
and the replay takes `apply_S` and the inverse blocks only.

lanczos_condition turns the PCG coefficients into the Lanczos tridiagonal T_k of the preconditioned operator M^-1 H
(Saad, "Iterative Methods for Sparse Linear Systems", section 6.7.3):
    T[j, j] = 1 / alpha_j + beta_{j-1} / alpha_{j-1},   T[j, j+1] = sqrt(beta_j) / alpha_j   (beta_0 = 0);
its extreme eigenvalues (Ritz values) approach those of M^-1 H from inside, so kappa = lmax / lmin is an estimate from below
of the condition number that governs how far PCG in finite precision strays from exact arithmetic.
"""
import numpy as np

NO_CONVERGENCE, SUCCESS, FAILURE = 0, 1, 2


def block_apply(inv_blocks, v):
    """y = M^-1 v for block-diagonal M^-1 given as [nc, 9, 9]"""
    return np.einsum("cij,cj->ci", inv_blocks, np.asarray(v, np.float64).reshape(-1, 9)).ravel()


def _preconditioner(inv_blocks):
    """M^-1 as a function: the [nc, 9, 9] inverse blocks, or any callable (a preconditioner of other block sizes)"""
    if callable(inv_blocks):
        return lambda v: np.asarray(inv_blocks(v), np.float64)
    blocks = np.asarray(inv_blocks, np.float64)
    return lambda v: block_apply(blocks, v)


def _zero_or_inf(v):
    return v == 0.0 or np.isinf(v)


def pcg_replay(apply_H, b, inv_blocks, *, eta, max_it, min_it=0, period=10):
    """The reference recurrence in float64 (inv_blocks: [nc, 9, 9] or a callable M^-1).  Returns a dict with
      xs       [x_0 = 0, x_1, ..., x_n]: every iterate (x_i after iteration i, including the residual refresh)
      zetas    zeta_i of iterations 1..n (index i - 1)
      alphas   alpha_i of iterations 1..n
      betas    beta_i = rho_{i+1} / rho_i, used to form p_{i+1} (index i - 1), of the iterations that formed one
      termination, iterations, num_matvecs (operator applications, the refreshes included)"""
    b = np.asarray(b, np.float64)
    Minv = _preconditioner(inv_blocks)
    H = (lambda v: np.asarray(apply_H(v), np.float64))
    out = {"xs": [np.zeros_like(b)], "zetas": [], "alphas": [], "betas": [], "termination": NO_CONVERGENCE,
           "iterations": 0, "num_matvecs": 0}
    norm_b = np.linalg.norm(b)
    if norm_b == 0.0:
        out["termination"] = SUCCESS
        return out
    x = np.zeros_like(b)
    r = b.copy()  # b - H x_0 with x_0 = 0 (the reference applies H to the zero vector)
    rho = 1.0
    q0 = -(x @ (b + r))
    p = None
    i = 1
    while True:
        z = Minv(r)
        last_rho = rho
        rho = r @ z
        if _zero_or_inf(rho):
            out["termination"] = FAILURE
            break
        if i == 1:
            p = z.copy()
        else:
            beta = rho / last_rho
            if _zero_or_inf(beta):
                out["termination"] = FAILURE
                break
            out["betas"].append(beta)
            p = z + beta * p
        q = H(p)
        out["num_matvecs"] += 1
        pq = p @ q
        if pq <= 0 or np.isinf(pq):
            out["termination"] = NO_CONVERGENCE
            break
        alpha = rho / pq
        if np.isinf(alpha):
            out["termination"] = FAILURE
            break
        out["alphas"].append(alpha)
        x = x + alpha * p
        if i % period == 0:
            r = b - H(x)
            out["num_matvecs"] += 1
        else:
            r = r - alpha * q
        out["xs"].append(x.copy())
        out["iterations"] = i
        q1 = -(x @ (b + r))
        zeta = i * (q1 - q0) / q1
        out["zetas"].append(zeta)
        if zeta < eta and i >= min_it:
            out["termination"] = SUCCESS
            break
        q0 = q1
        if i >= max_it:
            break
        i += 1
    return out


def power_replay(apply_S, inv_blocks, b, *, order, eta):
    """The reference power series in float64.  Returns a dict with
      sums     [accum_0, ..., accum_n]: every partial sum (accum_i after term i; already the increment)
      zetas    zeta_i = i |tmp_i| / |accum_i| of terms 1..n (index i - 1), computed whatever eta is
      termination, iterations (the number of terms n)"""
    b = np.asarray(b, np.float64)
    Minv = _preconditioner(inv_blocks)
    tmp = Minv(-b)
    acc = tmp.copy()
    out = {"sums": [acc.copy()], "zetas": [], "termination": NO_CONVERGENCE, "iterations": order}
    for i in range(1, order + 1):
        tmp = tmp - Minv(np.asarray(apply_S(tmp), np.float64))  # Hpp_d^-1 E0 tmp
        acc = acc + tmp
        out["sums"].append(acc.copy())
        zeta = i * np.linalg.norm(tmp) / np.linalg.norm(acc)
        out["zetas"].append(zeta)
        if eta > 0 and zeta < eta:
            out["termination"] = SUCCESS
            out["iterations"] = i
            break
    return out


def lanczos_condition(alphas, betas):
    """(lmin, lmax): extreme Ritz values of the Lanczos tridiagonal built from k PCG coefficients alpha_1..alpha_k and
    beta_1..beta_{k-1}; an estimate of the extreme eigenvalues of M^-1 H"""
    a = np.asarray(alphas, np.float64)
    k = a.size
    bt = np.asarray(betas, np.float64)[:k - 1]
    diag = 1.0 / a
    diag[1:] += bt / a[:-1]
    off = np.sqrt(bt) / a[:-1]
    ev = np.linalg.eigvalsh(np.diag(diag) + np.diag(off, 1) + np.diag(off, -1))
    return float(ev[0]), float(ev[-1])
