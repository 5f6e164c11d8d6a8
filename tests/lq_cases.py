"""Problem and case builders, oracle runs and error families that several CPU and GPU test modules share (CPU only:
numpy, the oracle, the references)."""
import numpy as np

import gen
import hp_reference as hp
import lq_adjoint_ref as aref
import lq_factor_adjoint_ref as fadj
import lq_factor_tangent_ref as ftan
import lq_resolve_ref as rref
import lq_refine_ref as fref
import lq_tangent_ref as tref
from aligator_b200.lqr import LqrKnot
from oracle import gar_oracle as orc


def batch_records(probs, case):
    """Packed records of the problems `probs`: stage [B][N][srec] padded to the record length, term [B][trec],
    G0 [B][nc0 * nx] (column-major) and g0 [B][nc0].  case = (nx, nu, nc, nct, nc0, N)."""
    nx, nu, nc, nct, nc0, N = case
    _, srec = aref.stage_offsets(nx, nu, nc)
    B = len(probs)
    stage = np.zeros((B, N, srec))
    for b, p in enumerate(probs):
        for t in range(N):
            r = gen.stage_record(p.stages[t])
            stage[b, t, :r.size] = r
    term = np.stack([gen.term_record(p.stages[N]) for p in probs])
    G0 = np.stack([np.asarray(p.G0).ravel(order="F") for p in probs]).reshape(B, nc0 * nx)
    g0 = np.stack([np.asarray(p.g0) for p in probs]).reshape(B, nc0)
    return stage, term, G0, g0


def case_records(case, seed, B=2, mutate=None):
    """Records of B seeded problems with a general initial condition; `mutate` edits the problems first."""
    nx, nu, nc, nct, nc0, N = case
    probs = gen.general_initial_condition(gen.generate_batch(seed, B, N, nx, nu, nc, nct), nc0, seed)
    if mutate:
        probs = mutate(probs) or probs
    return batch_records(probs, case)


def factor_oracle(recs, case, mu):
    nx, nu, nc, nct, nc0, N = case
    B = recs[1].shape[0]
    bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, B, *[np.ascontiguousarray(a) for a in recs])
    bo.sweep(mu, nthreads=1)
    assert np.all(bo.status == 1)
    o = bo.get()
    return dict(ff=o["ff"], fb=o["fb"], vxx=o["Vxx"], vx=o["vx"], fft=o["ffT"], fbt=o["fbT"])


def run_oracle(recs, d6, mu):
    """The oracle's batched sweep: its outputs in hp_reference's keys.  mu: a number, or one per instance (one oracle
    sweep per instance)."""
    nx, nu, nc, nct, nc0, N = d6
    B = recs[1].shape[0]
    if np.ndim(mu):
        per = [run_oracle([a[b:b + 1] for a in recs], d6, m) for b, m in enumerate(mu)]
        return {k: np.concatenate([o[k] for o in per]) for k in per[0]}
    bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, B, *[np.ascontiguousarray(a) for a in recs])
    bo.sweep(mu, nthreads=1)
    assert np.all(bo.status == 1)  # the oracle reports 1 = ok
    return bo.get()


def oracle_solution(recs, d6, mu):
    return aref.oracle_dict(run_oracle(recs, d6, mu))


def run_solver(probs, dims, mueq, algorithm="serial"):
    """The oracle's outputs in the product's layouts: the batched serial solver, or per instance its restatement of
    the dense solver ('dense') or of the parallel solver with T legs ('legsT')."""
    nx, nu, nc, nct, N = dims
    if algorithm == "serial":
        stage, term, G0, g0 = gen.pack_problems(probs)
        bo = orc.BatchedOracle(nx, nu, nc, nct, probs[0].nc0, N, len(probs), stage, term, G0, g0)
        bo.sweep(mueq, nthreads=1)
        assert np.all(bo.status == 1)
        return bo.get()
    return hp.stack_solutions([oracle_instance(p, mueq, algorithm) for p in probs])


def oracle_instance(p, mueq, algorithm):
    N = p.horizon
    nu, nc = p.stages[0].nu, p.stages[0].nc
    if algorithm == "dense":
        q = p.copy()
        kt = q.stages[-1]
        k0 = LqrKnot(kt.nx, 0, kt.nc, 0)  # the dense solver's terminal knot has nx2 = 0 (tests/test_oracle_dense.py)
        k0.Q[:], k0.q[:], k0.C[:], k0.d[:] = kt.Q, kt.q, kt.C, kt.d
        q.stages[-1] = k0
        op = orc.OracleProblem(q)
        s = orc.RiccatiSolverDense(op)
    else:
        op = orc.OracleProblem(p.copy())
        s = orc.ParallelRiccatiSolver(op, int(algorithm[4:]), threaded=False)
    assert s.backward(mueq)
    sol = orc.OracleSolution(op)
    assert s.forward(sol)
    xs, us, vs, lb = sol.get()
    o = dict(xs=np.stack(xs), us=np.stack(us[:N]).reshape(N, nu), vs=np.stack(vs[:N]).reshape(N, nc), vsT=vs[N],
             lbd0=lb[0], lbdas=np.stack(lb[1:]))
    if algorithm == "dense":
        fs = [s.factor(t) for t in range(N + 1)]
        o.update(fb=np.stack([f["fb"][:nu + nc] for f in fs[:N]]), ff=np.stack([f["ff"][:nu + nc] for f in fs[:N]]),
                 Vxx=np.stack([f["Pxx"] for f in fs]), vx=np.stack([f["px"] for f in fs]),
                 fbT=fs[N]["fb"][:p.stages[N].nc], ffT=fs[N]["ff"][:p.stages[N].nc])
    return o


TRAJ = ("xs", "us", "vs", "lbd")


def families(prog):
    """The families a program is measured on: leg mode's gains are parametric in the next leg's head and the dense
    program's rows after Z are its own (co-state, then closed loop), so those are measured on what they share."""
    if prog[0] == "legs":
        return TRAJ
    if prog[0] == "dense":
        return ("K", "k", "Z", "z", "Vxx", "vx") + TRAJ
    return hp.FAMILIES


def make_problem(seed, N, nx, nu, nc, nct, nth, gv=False):
    """A seeded parametric problem with non-trivial Gx, Gu, Gth and gamma on every knot.  Gv is zero unless `gv`:
    then Gaussian on every knot with rows (the terminal one included), drawn after everything else so the other
    blocks are those of gv=False.  (The reference's recursion is the exact theta-derivative only where Gv = 0,
    DESIGN §4; legs always have Gv = 0.)"""
    rng = np.random.default_rng(seed)
    x0 = rng.standard_normal(nx)
    p = gen.generate_lq_problem(rng, x0, N, nx, nu, nth, nc, singular=False, conditioned=True,
                                control_rows=nc > 0, term_nc=nct)
    for k in p.stages:  # non-trivial parametric blocks everywhere
        k.Gx[...] = 0.3 * rng.standard_normal(k.Gx.shape)
        k.Gu[...] = 0.3 * rng.standard_normal(k.Gu.shape)
        k.Gv[...] = 0.0
        g = rng.standard_normal((nth, nth))
        k.Gth[...] = g @ g.T / max(nth, 1) + np.eye(nth)
        k.gamma[...] = rng.standard_normal(nth)
    if gv:
        for k in p.stages:
            k.Gv[...] = rng.standard_normal(k.Gv.shape)
    return p


# ---------------------------------------------------------------------------------------------------------------------
# Parametric problems and leg mode at the level-2 bar
# ---------------------------------------------------------------------------------------------------------------------
# name: ((nx, nu, nc, nct, nth, N), batch, mueq, Gv != 0, nc0 of a Gaussian G0 (None: G0 = -I), theta scale)
PARAM_CASES = {
    "c3_mu1e-3": ((4, 2, 2, 0, 4, 20), 3, 1e-3, False, None, 1.0),
    "c3_mu1e-8": ((4, 2, 2, 0, 4, 20), 3, 1e-8, False, None, 1.0),
    "c3_gv": ((4, 2, 2, 0, 3, 12), 3, 1e-3, True, None, 1.0),
    "nct_gv": ((4, 2, 2, 2, 3, 10), 2, 1e-3, True, None, 1.0),
    "nth1": ((6, 3, 0, 0, 1, 8), 2, 1e-8, False, None, 1.0),
    "nth_nx": ((6, 3, 0, 0, 6, 8), 2, 1e-8, False, None, 1.0),
    "nth33": ((5, 2, 1, 0, 33, 4), 2, 1e-3, True, None, 1.0),
    "N0": ((4, 2, 2, 2, 3, 0), 2, 1e-3, True, None, 1.0),
    "N1": ((5, 2, 1, 0, 3, 1), 2, 1e-3, True, None, 1.0),
    "theta1e6": ((6, 3, 1, 0, 4, 8), 2, 1e-3, True, None, 1e6),
}
for _nc0 in (0, 1, 3, 6):
    PARAM_CASES["G0_nc0_%d" % _nc0] = ((6, 3, 1, 0, 3, 6), 2, 1e-3, True, _nc0, 1.0)


def param_problems(name, B=None, seed=0):
    """The problems and thetas [B][nth] of a parametric case (B instances, each its own problem and theta)."""
    (nx, nu, nc, nct, nth, N), B0, mueq, gv, nc0, scale = PARAM_CASES[name]
    B = B0 if B is None else B
    base = 5000 + 100 * seed + sum(map(ord, name))
    probs = [make_problem([base, b], N, nx, nu, nc, nct, nth, gv) for b in range(B)]
    if nc0 is not None:
        gen.general_initial_condition(probs, nc0, base)
    thetas = scale * np.random.default_rng(base).standard_normal((B, nth))
    return probs, thetas


def oracle_parametric(probs, mueq, thetas):
    """The oracle's ProximalRiccatiSolver on each problem, forward at its theta -> the outputs in hp_reference's
    keys and the product's layouts (those of hp_reference.solve_parametric).  mueq: a number or one per instance."""
    mus = np.broadcast_to(np.asarray(mueq, dtype=np.float64), (len(probs),))
    per = []
    for p, mu, th in zip(probs, mus, thetas):
        N = p.horizon
        nu, ncs = (p.stages[0].nu, p.stages[0].nc) if N else (0, 0)
        op = orc.OracleProblem(p)
        s = orc.ProximalRiccatiSolver(op)
        assert s.backward(mu)
        sol = orc.OracleSolution(op)
        assert s.forward(sol, th)
        fs = [s.factor(t) for t in range(N + 1)]
        k0 = s.kkt0()
        xs, us, vs, lb = sol.get()
        nr, nc, nth = fs[0]["fb"].shape[0], len(vs[0]), len(th)
        nct = fs[N]["fb"].shape[0] - fs[N]["dims"][1] - fs[N]["dims"][3]
        stk = lambda lst, *shape: np.stack(lst) if lst else np.zeros(shape)
        per.append(dict(fb=stk([f["fb"] for f in fs[:N]], 0, nr, len(xs[0])), ff=stk([f["ff"] for f in fs[:N]], 0, nr),
                        fth=stk([f["fth"] for f in fs[:N]], 0, nr, nth),
                        Vxx=np.stack([f["Vxx"] for f in fs]), vx=np.stack([f["vx"] for f in fs]),
                        Vxt=np.stack([f["Vxt"] for f in fs]), Vtt=np.stack([f["Vtt"] for f in fs]),
                        vt=np.stack([f["vt"] for f in fs]), fbT=fs[N]["fb"][:nct], ffT=fs[N]["ff"][:nct],
                        kkt0=k0["ff"], kkt0fth=k0["fth"], thGrad=k0["thGrad"], thHess=k0["thHess"],
                        xs=np.stack(xs), us=stk(us[:N], 0, nu).reshape(N, nu),
                        vs=stk(vs[:N], 0, ncs).reshape(N, ncs), vsT=vs[N], lbd0=lb[0],
                        lbdas=stk(lb[1:], 0, len(xs[0]))))
    return hp.stack_solutions(per)


def oracle_legs(probs, mueq, T):
    """The oracle's ParallelRiccatiSolver with T legs on each problem -> its factors in the product's layouts (leg
    mode: nth = nx, zero on the knots without parameters), its rollout, and `collapse`: the first gain after
    collapseFeedback."""
    per = []
    for p in probs:
        N, nx, nu = p.horizon, p.stages[0].nx, p.stages[0].nu
        op = orc.OracleProblem(p.copy())
        s = orc.ParallelRiccatiSolver(op, T, threaded=False)
        assert s.backward(mueq)
        sol = orc.OracleSolution(op)
        assert s.forward(sol)
        fs = [s.factor(t) for t in range(N + 1)]
        par = lambda f, k, *shape: f[k] if f["dims"][4] else np.zeros(shape)
        xs, us, vs, lb = sol.get()
        nr = fs[0]["fb"].shape[0]
        s.collapseFeedback()
        per.append(dict(fb=np.stack([f["fb"] for f in fs[:N]]), ff=np.stack([f["ff"] for f in fs[:N]]),
                        fth=np.stack([par(f, "fth", nr, nx) for f in fs[:N]]),
                        Vxx=np.stack([f["Vxx"] for f in fs]), vx=np.stack([f["vx"] for f in fs]),
                        Vxt=np.stack([par(f, "Vxt", nx, nx) for f in fs]),
                        Vtt=np.stack([par(f, "Vtt", nx, nx) for f in fs]), vt=np.stack([par(f, "vt", nx) for f in fs]),
                        fbT=fs[N]["fb"][:p.stages[N].nc], ffT=fs[N]["ff"][:p.stages[N].nc], xs=np.stack(xs), us=np.stack(us[:N]).reshape(N, nu),
                        vs=np.stack(vs[:N]).reshape(N, p.stages[0].nc), vsT=vs[N], lbd0=lb[0],
                        lbdas=np.stack(lb[1:]), collapse=s.factor(0)["fb"][:nu]))
    return hp.stack_solutions(per)


def param_oracle_errors(probs, mueq, thetas, ref):
    """e_oracle of parametric problems against the restatement's fp64 outputs `ref`: the error families of the oracle's
    ProximalRiccatiSolver, and on the theta-free factor families (K, k, Z, z, Vxx, vx) the larger of that and the
    oracle's dense solver's on the same problems without parameters.  Both are correct fp64 solvers; where a quantity
    comes out of a cancellation (z = (d + D k) / mu on an active row, say) one of them alone can land unrepresentatively
    close, as in tests/test_hp_emulation.py's bar for the dense and leg programs."""
    nx, nu, nc, nct, nc0, N = hp.dims_of(probs[0])
    e = hp.error_families(oracle_parametric(probs, mueq, thetas), ref, nu, nc, N)
    if N == 0:
        return e
    plain = []
    for p in probs:
        q = p.copy()
        q.addParameterization(0)
        plain.append(q)
    dense = hp.error_families(run_solver(plain, (nx, nu, nc, nct, N), mueq, "dense"), ref, nu, nc, N,
                              ("K", "k", "Z", "z", "Vxx", "vx"))
    return {f: max(v, dense.get(f, 0.0)) for f, v in e.items()}


PARAM_KEYS = ("fth", "Vxt", "Vtt", "vt", "kkt0fth", "thGrad", "thHess")
LEG_FAMILIES = ("K", "k", "Z", "z", "Ahat", "a", "Vxx", "vx", "Kth", "Zth", "Yth", "Vxt", "Vtt", "vt", "collapse")


def symmetric_dot(rng, d6, B):
    """A data tangent in the records' layouts with symmetric Q, R and Q_N (the pad double random too)."""
    nx, nu, nc, nct, nc0, N = d6
    so, srec = aref.stage_offsets(nx, nu, nc)
    to, trec = aref.term_offsets(nx, nct)
    dot = dict(stage=rng.standard_normal((B, N, srec)), term=rng.standard_normal((B, trec)),
               G0=rng.standard_normal((B, nc0 * nx)), g0=rng.standard_normal((B, nc0)))
    for key, off, k in (("stage", so["Q"], nx), ("stage", so["R"], nu), ("term", to["Q"], nx)):
        x = dot[key]
        M = x[..., off[0]:off[1]].reshape(*x.shape[:-1], k, k)
        x[..., off[0]:off[1]] = (M + np.swapaxes(M, -1, -2)).reshape(*x.shape[:-1], k * k)
    return dot


class Case:
    """One case's problems, the oracle's outputs, the inputs of every derivative call, the extended-precision
    references (fp64-rounded) and the fp64 restatements' results fed by the oracle."""

    def __init__(self, probs, mu, seed=1, inputs=None):
        """inputs: the cotangents and the tangent (cot, fcot, dot) to use instead of random ones."""
        self.probs, self.mu = probs, mu
        self.d6 = hp.dims_of(probs[0])
        B = len(probs)
        self.recs = hp.records(probs)
        rng = np.random.default_rng(seed)
        if inputs is None:
            inputs = dict(cot={k: rng.standard_normal(s) for k, s in aref._shapes(self.d6, B).items()},
                          fcot=fadj.random_cot(rng, self.d6, B), dot=symmetric_dot(rng, self.d6, B))
        self.cot, self.fcot, self.dot = inputs["cot"], inputs["fcot"], inputs["dot"]
        # extended precision
        _, self.hps = hp.solve(probs, mu)
        self.g_hp = hp.grads64(hp.grad_solution(probs, mu, self.cot, self.hps))
        self.gf_hp = hp.grads64(hp.grad_factor(probs, mu, self.fcot, self.hps))
        td, _ = hp.tangents(probs, mu, self.dot)
        self.zd_hp, self.fd_hp = hp.solution_of(td), hp.factor_of(td)
        # the oracle and the fp64 restatements fed by it
        self.out = run_oracle(self.recs, self.d6, mu)
        self.z, self.fac = aref.oracle_dict(self.out), hp.factor_of(self.out)
        w = oracle_solution(aref.adjoint_records(*self.recs, self.cot, self.d6), self.d6, mu)
        self.g_ref = aref.grad_records(self.z, w, self.d6)
        self.zd_ref = oracle_solution(tref.tangent_records(*self.recs, self.dot, self.z, self.d6), self.d6, mu)
        f = self.fac
        self.gf_ref = fadj.factor_adjoint(self.recs[0], self.recs[1], f["ff"], f["fb"], f["vxx"], f["vx"], f["fft"],
                                          f["fbt"], self.fcot, self.d6, mu)
        self.fd_ref = ftan.factor_tangent(self.recs[0], self.recs[1], f["ff"], f["fb"], f["vxx"], f["vx"], f["fft"],
                                          f["fbt"], self.dot, self.d6, mu)

    # the error families of each call's output against the reference
    def e_adjoint(self, g):
        return hp.grad_errors(g, self.g_hp, self.d6)

    def e_tangent(self, zd):
        return hp.solution_errors(zd, self.zd_hp, self.d6)

    def e_factor_adjoint(self, g):
        return hp.grad_errors(g, self.gf_hp, self.d6, hp.GRAD_FAMILIES[:-2])

    def e_factor_tangent(self, fd):
        return hp.factor_errors(fd, self.fd_hp, self.d6)

    def e_refs(self):
        return dict(adjoint=self.e_adjoint(self.g_ref), tangent=self.e_tangent(self.zd_ref),
                    factor_adjoint=self.e_factor_adjoint(self.gf_ref),
                    factor_tangent=self.e_factor_tangent(self.fd_ref))

    def e_torch(self):
        """The fp64 torch derivation's errors on the factorisation's derivatives (autograd and jvp through
        lq_factor_adjoint_ref.torch_factor)."""
        st, tt = self.recs[0], self.recs[1]
        B = tt.shape[0]
        mus = np.broadcast_to(np.asarray(self.mu, dtype=np.float64), (B,))
        one = lambda d, b: {k: v[b:b + 1] for k, v in d.items()}
        per = [(fadj.autograd(st[b:b + 1], tt[b:b + 1], self.d6, mus[b], one(self.fcot, b))[1],
                ftan.jvp(st[b:b + 1], tt[b:b + 1], self.d6, mus[b],
                         dict(stage=self.dot["stage"][b:b + 1], term=self.dot["term"][b:b + 1]))[1]) for b in range(B)]
        ga, jv = ({k: np.concatenate([p[i][k] for p in per]) for k in per[0][i]} for i in (0, 1))
        ga.update(G0=np.zeros((B, self.d6[4] * self.d6[0])), g0=np.zeros((B, self.d6[4])))
        return dict(factor_adjoint=self.e_factor_adjoint(ga), factor_tangent=self.e_factor_tangent(jv))


def check_bar(e_kernel, e_ref, title, e_torch=None):
    """e_kernel <= max(16 e_ref, 64 u) family by family; the table of the case on failure."""
    bad = hp.violations(e_kernel, e_ref)
    assert not bad, hp.table(title, e_ref, e_kernel, e_torch)


def block_errors(got, want, case):
    """Relative Frobenius error of every record block (gradient family) of the stage and terminal records."""
    nx, nu, nc, nct, nc0, N = case
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    errs = {}
    for name, off, key in [(k, v, "stage") for k, v in so.items()] + [("N" + k, v, "term") for k, v in to.items()]:
        w = want[key][..., off[0]:off[1]]
        if w.size:
            e = gen.rel_fro(got[key][..., off[0]:off[1]], w)
            errs[name] = e if np.isfinite(e) else np.inf  # an entry left unwritten fails
    return errs


def family_errors(got, want):
    """Relative Frobenius error of every output family of nonzero size."""
    errs = {}
    for k in fadj.COT:
        w = np.asarray(want[k])
        if w.size:
            e = gen.rel_fro(got[k], w)
            errs[k] = e if np.isfinite(e) else np.inf  # an entry left unwritten fails
    return errs


def device_cot(cot, case, B):
    """Restatement-shaped cotangents -> the device layouts (vxx column-major per block); None stays None."""
    out = {}
    for k, v in cot.items():
        if v is None:
            out[k] = None
        elif k == "vxx":
            out[k] = np.ascontiguousarray(np.swapaxes(v, -1, -2))
        else:
            out[k] = np.ascontiguousarray(v)
    return out


def random_dot(rng, case, B):
    """Tangent records with every entry random: Q, R and Q_N asymmetric, the pad double too."""
    nx, nu, nc, nct, nc0, N = case
    _, srec = aref.stage_offsets(nx, nu, nc)
    _, trec = aref.term_offsets(nx, nct)
    return dict(stage=rng.standard_normal((B, N, srec)), term=rng.standard_normal((B, trec)))


def out_shapes(case, B):
    nx, nu, nc, nct, nc0, N = case
    nr = nu + nc + nx
    return dict(ff=(B, N, nr), fb=(B, N, nr, nx), vxx=(B, N + 1, nx, nx), vx=(B, N + 1, nx), fft=(B, nct),
                fbt=(B, nct, nx))


def cot_rhs(c):
    """A cotangent as resolve's right-hand side: xs -> q, us -> r, vs -> d, vsT -> dN, lam0 -> g0, lams -> f."""
    return dict(q=c["xs"], r=c["us"], d=c["vs"], dN=c["vsT"], g0=c["lam0"], f=c["lams"])


# name: ((nx, nu, nc, nct, N), B, mu, transform)
BAR_CASES = {
    "c3_mu1e-3": ((4, 2, 2, 0, 20), 3, 1e-3, None),
    "c3_mu1e-8": ((4, 2, 2, 0, 30), 3, 1e-8, None),
    "c3_mu1e-11": ((4, 2, 2, 0, 30), 3, 1e-11, None),
    "c3_nct_mu1e-8": ((4, 2, 2, 2, 10), 2, 1e-8, None),
    "pivots_2x2_mu1e-3": ((4, 2, 2, 0, 10), 2, 1e-3, gen.make_2x2_pivots),
    "pivots_2x2_mu1e-8": ((4, 2, 2, 0, 10), 2, 1e-8, gen.make_2x2_pivots),
    "interchanges": ((12, 6, 0, 0, 8), 2, 1e-8, gen.make_pivoting),
}


def bar_case(name):
    """(problems, packed records, dims, mu, right-hand sides [2][B][...])."""
    (nx, nu, nc, nct, N), B, mu, transform = BAR_CASES[name]
    probs = gen.generate_batch(3000 + sum(map(ord, name)), B, N, nx, nu, nc, nct)
    if transform is not None:
        transform(probs)
    case = (nx, nu, nc, nct, nx, N)
    return probs, batch_records(probs, case), case, mu, rref.random_rhs(np.random.default_rng(len(name)), case, B, 2)


def bar_violations(probs, recs, case, mu, hj, got):
    """Families of the trajectory where `got` (one right-hand side's solution dict) is further from the extended-precision
    solve of the replaced problem than max(16 e_oracle, 64 u) allows."""
    nx, nu, nc, nct, nc0, N = case
    want, _ = hp.solve(rref.replaced_problems(probs, hj), mu)
    e_oracle = hp.error_families(run_oracle(rref.replaced_records(*recs, hj, case), case, mu), want, nu, nc, N, TRAJ)
    z = dict(got, lbd0=got["lam0"], lbdas=got["lams"])
    e_kernel = hp.error_families(z, want, nu, nc, N, TRAJ)
    return hp.violations(e_kernel, e_oracle), hp.table("", e_oracle, e_kernel)


def refine_case(name):
    """(problems, records, dims, mu) of a refinement case: the conditioning-bar cases of the resolve tests and a
    general G0."""
    if name == "general_G0":
        probs = gen.general_initial_condition(gen.generate_batch(4100, 3, 20, 4, 2, 2, 0), 2, 4100)
        case, mu = (4, 2, 2, 0, 2, 20), 1e-8
    else:
        (nx, nu, nc, nct, N), B, mu, transform = BAR_CASES[name]
        probs = gen.generate_batch(3000 + sum(map(ord, name)), B, N, nx, nu, nc, nct)
        if transform is not None:
            transform(probs)
        case = (nx, nu, nc, nct, nx, N)
    return probs, batch_records(probs, case), case, mu


def errors(z, want, case):
    """Error families (xs, us, vs, lbd) of right-hand side 0 of the solution dict z against hp_reference's `want`."""
    nx, nu, nc, nct, nc0, N = case
    got = {k: v[0] for k, v in z.items()}
    return hp.error_families(dict(got, lbd0=got["lam0"], lbdas=got["lams"]), want, nu, nc, N, ("xs", "us", "vs", "lbd"))


def refined_on_oracle(probs, recs, case, mu, steps=2):
    """(refined z, unrefined z, norms, extended-precision solution, floor) for the primal of `probs`, refined on the
    oracle's factorisation.  floor: per family, the larger error after one and after two steps started from the
    correctly rounded solution -- the noise level of a refinement whose residual is computed in fp64."""
    o = run_oracle(recs, case, mu)
    fac = (o["fb"], o["fbT"], o["Vxx"])
    z0 = {k: v[None] for k, v in aref.oracle_dict(o).items()}
    z, norms = fref.refine(*recs, *fac, z0, None, case, mu, steps)
    want, _ = hp.solve(probs, mu)
    exact = {k: want[w][None] for k, w in zip(aref.KEYS, ("xs", "us", "vs", "vsT", "lbd0", "lbdas"))}
    e1 = errors(fref.refine(*recs, *fac, exact, None, case, mu, 1)[0], want, case)
    e2 = errors(fref.refine(*recs, *fac, exact, None, case, mu, 2)[0], want, case)
    return z, z0, norms, want, {f: max(e1[f], e2[f]) for f in e1}


def jacobian_records(case, seed):
    """case_records of a (nx, nu, nc, nct, nc0, N, B) case."""
    return case_records(case[:6], seed, case[6])


# (nx, nu, nc, nct, nc0, N): C1, C2 and C3 dims, nc > 0, nct > 0, horizon 0 and 1
FACTOR_CASES = [(6, 3, 0, 0, 6, 4), (6, 3, 0, 2, 3, 1), (12, 6, 0, 0, 12, 3), (12, 6, 0, 3, 1, 0), (4, 2, 2, 2, 4, 5),
                (4, 2, 2, 0, 0, 1), (4, 2, 2, 2, 2, 0), (5, 2, 1, 1, 0, 3)]
FACTOR_IDS = ["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d" % c for c in FACTOR_CASES]
