"""CPU restatement (numpy) of the rest of SolverProxDDP's inner iteration -- TEST INFRASTRUCTURE ONLY, never imported
by the product.  For ONE problem instance, statement by statement:

  computeMultipliers              solvers/proxddp/solver-proxddp.hxx:220-318
  LagrangianDerivatives::compute  core/lagrangian.hpp:29-92
  computeCriterion                solvers/proxddp/solver-proxddp.hxx:703-732
  normalConeProjection            equality-constraint.hpp:37-40, negative-orthant.hpp:36-38, box-constraint.hpp:27-37

Per-knot data are lists indexed by the knot: xs, lams, vs, prev_vs, cvals hold N+1 vectors (lams[0] = the initial
condition's multiplier, vs[N] / cvals[N] the terminal constraints, empty when there are none).  Constraint sets are
given per row by the bounds of include/aligator_b200/gar.h (equality rows: lo = +inf).

PARITY UNPINNED: the reference cannot be built here (no Eigen); the restatement is checked against hand-computed
numbers and an independent dense formulation in tests/test_proxddp_inner.py.
"""
import numpy as np


def normal_cone(z, lo, hi):
    """Row-wise projection onto the normal cone: z on equality rows, z - max(min(z, hi), lo) elsewhere."""
    eq = lo == np.inf
    with np.errstate(invalid="ignore"):
        box = z - np.maximum(np.minimum(z, hi), lo)
    return np.where(eq, z, box)


def compute_multipliers(xs, lams, vs, prev_vs, init_value, cvals, lo, hi, loN, hiN, mu, mu_dyn, xnext=None, fs=None):
    """-> dict fs (N+1: fs[0] = init_value), lams_plus (N+1), vs_plus, shifted, Lvs, stage_infeas (N+1 each; the
    terminal entries are empty without terminal constraints), prim_infeas and ok.  `xnext` (N vectors, vector-space
    difference) or `fs` (N vectors = fs[1..N]).  Restated without the early returns: ok is what RET_FALSE_IF_NAN
    would have returned, every output is computed."""
    N = len(xs) - 1
    mu_inv = 1.0 / mu                                                  # mu_inv()
    fsl = [None] * (N + 1)
    lams_plus, vs_plus = [None] * (N + 1), [None] * (N + 1)
    shifted, Lvs, infeas = [None] * (N + 1), [None] * (N + 1), [None] * (N + 1)
    ok = True
    fsl[0] = np.array(init_value, dtype=np.float64)                   # :246
    lams_plus[0] = lams[0] + fsl[0] / mu                              # :247 (mu, not mu_dyn)
    ok &= bool(np.all(np.isfinite(lams_plus[0])))                     # :248
    for i in range(N):
        fsl[i + 1] = (xnext[i] - xs[i + 1]) if fs is None else np.array(fs[i])   # :263 difference(x_{i+1}, xnext)
        lams_plus[i + 1] = lams[i + 1] + fsl[i + 1] / mu_dyn          # :264
        ok &= bool(np.all(np.isfinite(lams_plus[i + 1])))             # :265
        shifted[i] = cvals[i] + mu * prev_vs[i]                       # :275-277
        nc = normal_cone(shifted[i], lo, hi)                          # :278
        Lvs[i] = nc - mu * vs[i]                                      # :281-282
        vs_plus[i] = mu_inv * nc                                      # :283
        infeas[i] = mu * (vs_plus[i] - prev_vs[i])                    # :286
        ok &= bool(np.all(np.isfinite(Lvs[i])))                       # :289
    if len(cvals[N]) > 0:                                             # :292
        shifted[N] = cvals[N] + mu * prev_vs[N]                       # :296-301
        nc = normal_cone(shifted[N], loN, hiN)                        # :302
        Lvs[N] = nc - mu * vs[N]                                      # :305-306
        vs_plus[N] = mu_inv * nc                                      # :307
        infeas[N] = mu * (vs_plus[N] - prev_vs[N])                    # :310
        ok &= bool(np.all(np.isfinite(Lvs[N])))                       # :313
    else:
        shifted[N] = vs_plus[N] = Lvs[N] = infeas[N] = np.zeros(0)
    inf_norm = lambda vs_: max([float(np.max(np.abs(v))) if len(v) else 0.0 for v in vs_] + [0.0])  # math::infty_norm
    prim = max(inf_norm(infeas), inf_norm(fsl))                       # :315-316
    return dict(fs=fsl, lams_plus=lams_plus, vs_plus=vs_plus, shifted=shifted, Lvs=Lvs, stage_infeas=infeas,
                prim_infeas=prim, ok=ok)


def lagrangian_gradient(lx, lu, lx_N, Jx, Ju, cJx, cJu, cJx_N, G0, lams, vs, force_initial_condition=False):
    """-> (Lxs: N+1 vectors, Lus: N vectors).  Stage lists lx, lu, Jx, Ju, cJx, cJu have N entries (matrices as
    numpy 2-D arrays, rows = function outputs); lams, vs have N+1.  force_initial_condition applies innerLoop's
    Lxs[0].setZero() (solver-proxddp.hxx:592-594)."""
    N = len(lx)
    nx = len(lx_N)
    Lxs = [np.zeros(nx) for _ in range(N + 1)]                        # :47 setZero
    Lus = [np.zeros(len(lu[i])) for i in range(N)]                    # :48
    Lxs[0] = G0.T @ lams[0]                                           # :52-53
    for i in range(N):
        Lxs[i] = Lxs[i] + lx[i]                                       # :60
        Lus[i] = lu[i].copy()                                         # :61
        Lxs[i] = Lxs[i] + Jx[i].T @ lams[i + 1]                       # :63
        Lus[i] = Lus[i] + Ju[i].T @ lams[i + 1]                       # :64
        Lxs[i] = Lxs[i] + cJx[i].T @ vs[i]                            # :70 (one stacked constraint block)
        Lus[i] = Lus[i] + cJu[i].T @ vs[i]                            # :71
        Lxs[i + 1] = -lams[i + 1]                                     # :75
    Lxs[N] = Lxs[N] + lx_N                                            # :84
    Lxs[N] = Lxs[N] + cJx_N.T @ vs[N]                                 # :89
    if force_initial_condition:
        Lxs[0] = np.zeros(nx)
    return Lxs, Lus


def criterion(Lxs, Lus, fs, Lvs):
    """-> (inner_criterion, dual_infeas).  fs: N+1 dynamics slacks (fs[0] = initial residual), Lvs: N+1 (the
    terminal entry empty without terminal constraints)."""
    N = len(Lus)
    n = lambda v: float(np.max(np.abs(v))) if len(v) else 0.0        # math::infty_norm
    crits, xdual, udual = [], [], []
    for i in range(N):
        rx, ru, rd, rc = n(Lxs[i]), n(Lus[i]), n(fs[i]), n(Lvs[i])  # :712-717 (stage i's residual is fs[i])
        crits.append(max(rx, ru, rd, rc))                             # :719
        xdual.append(rx)
        udual.append(ru)
    rx, rc = n(Lxs[N]), n(Lvs[N])                                     # :723-724
    xdual.append(rx)
    crits.append(max(rx, rc))                                         # :726
    return max(crits), max(max(xdual), max(udual + [0.0]))           # :728-731
