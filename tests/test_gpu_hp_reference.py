"""The CUDA sweep programs against the extended-precision restatement of the sweep (tests/hp_reference.py), with the
conditioning-aware tolerance of tests/test_hp_emulation.py: e_kernel <= max(16 e_oracle, 64 u) for every family.
Also on the device: general initial conditions, homogeneous problems, exact per-instance rescaling through the *_v
twins, and ab2_gar_kkt_error against residuals evaluated exactly (fractions.Fraction) from the same fp64 data."""
import functools
from fractions import Fraction

import numpy as np
import pytest

import gen
import hp_reference as hp
from lq_cases import families, run_solver

pytestmark = pytest.mark.gpu

VARIANTS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 10]


@pytest.fixture(scope="module")
def gar():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    return gar


def run_cuda(gar, probs, dims, mueq, prog=("default", -1, 0), kkt=False):
    """prog = (kind, variant, legs), kind in default / variant / dense / legs.  Outputs in the oracle's shapes."""
    kind, variant, legs = prog
    nx, nu, nc, nct, N = dims
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, probs[0].nc0, N, len(probs), variant=variant, legs=legs,
                             dense=kind == "dense")
    s.set_problem(*gar.pack_problems(probs))
    s.sweep(mueq)
    out = {k: s.get(w).copy() for k, w in dict(
        ff=gar.OUT_FF, fb=gar.OUT_FB, Vxx=gar.OUT_VXX, vx=gar.OUT_VX, ffT=gar.OUT_FFT, fbT=gar.OUT_FBT,
        kkt0=gar.OUT_KKT0, xs=gar.OUT_XS, us=gar.OUT_US, vs=gar.OUT_VS, vsT=gar.OUT_VST, lbd0=gar.OUT_LBD0,
        lbdas=gar.OUT_LBDAS).items()}
    out["status"] = s.status().copy()
    if kkt:
        out["kkt"] = s.kkt_error(mueq)
    s.close()
    return out


# name: ((nx, nu, nc, nct, N), batch, mueq, transform, programs)
DEFAULT, CTA, DENSE = ("default", -1, 0), ("variant", 9, 0), ("dense", -1, 0)
LEGS = [("legs", -1, 2), ("legs", -1, 4)]
ALL_WARP = [("variant", v, 0) for v in VARIANTS] + [CTA]
CASES = {
    "c2": ((12, 6, 0, 0, 20), 5, 1e-8, None, [DEFAULT] + ALL_WARP + [DENSE] + LEGS),
    "c3": ((4, 2, 2, 0, 20), 9, 1e-3, None, [DEFAULT] + ALL_WARP + [DENSE] + LEGS),
    "c3_mu1e-8": ((4, 2, 2, 0, 100), 8, 1e-8, None, [DEFAULT, CTA, DENSE]),
    "c3_mu1e-11": ((4, 2, 2, 0, 100), 8, 1e-11, None, [DEFAULT, CTA, DENSE]),
    "nct": ((4, 2, 2, 3, 12), 5, 1e-3, None, [DEFAULT, CTA, DENSE]),
    "pivots_2x2": ((4, 2, 2, 0, 12), 5, 1e-3, gen.make_2x2_pivots, [DEFAULT, CTA]),
    "interchanges": ((12, 6, 0, 0, 10), 3, 1e-8, gen.make_pivoting, [DEFAULT, ("variant", 7, 0), CTA]),
    "cta_7_3_0": ((7, 3, 0, 0, 10), 3, 1e-8, None, [DEFAULT]),
    "cta_9_5_3": ((9, 5, 3, 0, 8), 3, 1e-3, None, [DEFAULT]),
    "cta_20_9_0": ((20, 9, 0, 0, 6), 2, 1e-8, None, [DEFAULT]),
    "cta_57_28_0": ((57, 28, 0, 0, 2), 1, 1e-8, None, [DEFAULT]),
}
for _dims, _mu in (((4, 2, 2, 2, 8), 1e-3), ((12, 6, 0, 0, 8), 1e-8), ((7, 3, 0, 0, 6), 1e-8)):
    for _nc0 in sorted({0, 1, _dims[0] // 2, _dims[0]}):
        CASES["G0_%d_nc0_%d" % (_dims[0], _nc0)] = (_dims, 3, _mu, ("G0", _nc0), [DEFAULT, CTA, DENSE, LEGS[0]])


def make_problems(name):
    dims, B, mueq, transform, _ = CASES[name]
    nx, nu, nc, nct, N = dims
    probs = gen.generate_batch(2000 + sum(map(ord, name)), B, N, nx, nu, nc, nct)
    if isinstance(transform, tuple):
        gen.general_initial_condition(probs, transform[1], 78)
    elif transform is not None:
        transform(probs)
    return probs


@functools.lru_cache(maxsize=None)
def case(name):
    dims, B, mueq, _, _ = CASES[name]
    probs = make_problems(name)
    ref, _ = hp.solve(probs, mueq)
    return probs, ref, hp.error_families(run_solver(probs, dims, mueq), ref, dims[1], dims[2], dims[4])


@functools.lru_cache(maxsize=None)
def oracle_errors(name, algorithm):
    """As tests/test_hp_emulation.py: for the dense and leg programs the larger of the serial oracle's error and that of
    the oracle's restatement of the same algorithm."""
    dims, B, mueq, _, _ = CASES[name]
    probs, ref, e = case(name)
    if algorithm == "serial":
        return e
    own = hp.error_families(run_solver(probs, dims, mueq, algorithm), ref, dims[1], dims[2], dims[4])
    return {f: max(v, e[f]) for f, v in own.items()}


def _emu_like(prog):
    """(kind, ...) in the shape tests/test_hp_emulation.py's families() expects."""
    return {"dense": ("dense", 1, False, 0), "legs": ("legs", 1, False, prog[2])}.get(prog[0], ("group", 0, False, 0))


def prog_id(p):
    return {"default": "default", "variant": "v%d" % p[1], "dense": "dense", "legs": "legs%d" % p[2]}[p[0]]


ITEMS = [(n, p) for n in CASES for p in CASES[n][4]]


@pytest.mark.parametrize("name,prog", ITEMS, ids=["%s-%s" % (n, prog_id(p)) for n, p in ITEMS])
def test_kernel_against_extended_precision(gar, name, prog):
    dims, B, mueq, _, _ = CASES[name]
    nx, nu, nc, nct, N = dims
    probs, ref, _ = case(name)
    got = run_cuda(gar, probs, dims, mueq, prog)
    assert np.all(got["status"] == 0), got["status"]
    em = _emu_like(prog)
    e_oracle = oracle_errors(name, {"dense": "dense", "legs": "legs%d" % prog[2]}.get(prog[0], "serial"))
    e_kernel = hp.error_families(got, ref, nu, nc, N, families(em))
    print("\n" + hp.table("%s %s" % (name, prog_id(prog)), e_oracle, e_kernel))
    bad = hp.violations(e_kernel, e_oracle)
    assert not bad, hp.table("%s %s" % (name, prog_id(prog)), e_oracle, e_kernel)


C2_SAMPLE = [0, 1, 2, 3, 263, 264, 527, 528, 1055, 1056, 2047, 2048, 4092, 4093, 4094, 4095]


def test_full_size_c2_sampled_instances(gar):
    """BASELINE config 2 at full size (the benchmark's inputs, nx12 nu6 N100, 4096 instances, mu = 1e-11): 16 instances
    from the first wave, across wave boundaries and from the ragged tail, against the extended-precision result."""
    import torch
    bench = __import__("bench")
    nx, nu, N, B, mueq = 12, 6, 100, 4096, 1e-11
    stage, term, G0, g0 = bench.synth_batch_torch(torch, B, N, nx, nu, torch.device("cuda:0"), 7, 0)
    # Q, R (and the terminal Q) exactly symmetric from their lower triangles, so that the problem is one symmetric LQ
    # problem whatever rounding the batched products that built them did
    st = stage.view(B, N, -1)
    for off, n in ((nx * nx + nx * nu + nx, nx), (2 * nx * nx + 2 * nx * nu + nx, nu)):  # [A|B|f|Q|S|R|q|r]
        M = st[..., off:off + n * n].reshape(B, N, n, n)
        st[..., off:off + n * n] = (M.tril() + M.tril(-1).transpose(-1, -2)).reshape(B, N, n * n)
    M = term[:, :nx * nx].reshape(B, nx, nx)
    term[:, :nx * nx] = (M.tril() + M.tril(-1).transpose(-1, -2)).reshape(B, nx * nx)
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
    s.sweep(mueq)
    assert np.all(s.status() == 0)
    idx = C2_SAMPLE
    got = {k: s.get(w)[idx] for k, w in dict(ff=gar.OUT_FF, fb=gar.OUT_FB, Vxx=gar.OUT_VXX, vx=gar.OUT_VX,
                                            ffT=gar.OUT_FFT, fbT=gar.OUT_FBT, xs=gar.OUT_XS, us=gar.OUT_US,
                                            vs=gar.OUT_VS, vsT=gar.OUT_VST, lbd0=gar.OUT_LBD0,
                                            lbdas=gar.OUT_LBDAS).items()}
    s.close()
    st, tm, g0m, g0v = (a.cpu().numpy() for a in (stage, term, G0, g0))
    probs = [unpack(st[b].reshape(N, -1), tm[b], g0m[b], g0v[b], nx, nu) for b in idx]
    ref, _ = hp.solve(probs, mueq)
    e_oracle = hp.error_families(run_solver(probs, (nx, nu, 0, 0, N), mueq), ref, nu, 0, N)
    e_kernel = hp.error_families(got, ref, nu, 0, N)
    print("\n" + hp.table("C2 full size, 16 sampled instances", e_oracle, e_kernel))
    assert not hp.violations(e_kernel, e_oracle), hp.table("C2", e_oracle, e_kernel)


def unpack(stage, term, G0, g0, nx, nu):
    """Packed records (include/aligator_b200/gar.h, nc = nct = 0) -> LqrProblem."""
    from aligator_b200.lqr import LqrKnot, LqrProblem
    knots = []
    for rec in stage:
        k = LqrKnot(nx, nu, 0)
        o = 0
        for name, shape in (("A", (nx, nx)), ("B", (nx, nu)), ("f", (nx,)), ("Q", (nx, nx)), ("S", (nx, nu)),
                            ("R", (nu, nu)), ("q", (nx,)), ("r", (nu,))):
            n = int(np.prod(shape))
            getattr(k, name)[...] = rec[o:o + n].reshape(shape, order="F")
            o += n
        knots.append(k)
    kt = LqrKnot(nx, 0, 0)
    kt.Q[...] = term[:nx * nx].reshape(nx, nx, order="F")
    kt.q[...] = term[nx * nx:nx * nx + nx]
    p = LqrProblem(knots + [kt], nx)
    p.G0[...] = G0.reshape(nx, nx, order="F")
    p.g0[...] = g0
    return p


# ---------------------------------------------------------------------------------------------------------------------
# Homogeneous problems, exact rescaling
# ---------------------------------------------------------------------------------------------------------------------
ZERO_KEYS = ("ff", "ffT", "xs", "us", "vs", "vsT", "lbd0", "lbdas")


@pytest.mark.parametrize("dims,nc0,progs", [
    ((4, 2, 2, 2, 8), 2, [DEFAULT] + ALL_WARP + [DENSE] + LEGS),
    ((12, 6, 0, 0, 8), 12, [DEFAULT] + ALL_WARP + [DENSE] + LEGS),
    ((9, 5, 3, 2, 6), 9, [DEFAULT, DENSE, LEGS[0]])])
def test_homogeneous_problem_has_exactly_zero_solution(gar, dims, nc0, progs):
    nx, nu, nc, nct, N = dims
    probs = gen.generate_batch(62, 37, N, nx, nu, nc, nct)
    if nc0 != nx:
        gen.general_initial_condition(probs, nc0, 3)
    gen.make_homogeneous(probs)
    for prog in progs:
        got = run_cuda(gar, probs, dims, 1e-3 if nc + nct else 1e-8, prog)
        assert np.all(got["status"] == 0), prog
        for k in ZERO_KEYS:
            assert np.all(got[k] == 0.0), (prog, k)
        assert np.all(np.isfinite(got["fb"])) and np.any(got["fb"] != 0), prog


EXACT = ("ff", "fb", "ffT", "fbT", "xs", "us", "vs", "vsT", "lbd0", "kkt0")
SCALED = ("Vxx", "vx", "lbdas")
EXPONENTS = (-60, 0, 37, 60, -23, 11, -1, 45, -52)


@pytest.mark.parametrize("dims,nc0,progs", [
    ((12, 6, 0, 0, 10), 12, [DEFAULT] + ALL_WARP),
    ((12, 6, 0, 0, 10), 6, [DEFAULT, ("variant", 7, 0), CTA]),
    ((4, 2, 2, 2, 10), 2, [DEFAULT] + ALL_WARP),
    ((4, 2, 2, 0, 10), 4, [DEFAULT, ("variant", 1, 0), CTA]),
    ((7, 3, 0, 2, 6), 7, [DEFAULT]),
    ((9, 5, 3, 0, 6), 4, [DEFAULT]),
])
def test_exact_per_instance_rescaling(gar, dims, nc0, progs):
    """Instance b scaled by c_b = 2**s_b (s_b in [-60, 60]) with mu_b = c_b mu through sweep_v / kkt_error_v: fb, ff,
    xs, us, vs, lbd0 bit for bit those of the unscaled batch; Vxx, vx, lbdas and columns 2, 3 of kkt_error c_b times
    them.  More instances than exponents, so the scaled instances share warps, sub-warp groups and CTAs with unscaled
    ones.  Not leg mode (absolute refinement threshold) nor the dense program (its stage system is not c_b times the
    original, see tests/test_hp_emulation.py)."""
    nx, nu, nc, nct, N = dims
    B = 3 * len(EXPONENTS)
    probs = gen.generate_batch(72, B, N, nx, nu, nc, nct)
    if nc0 != nx:
        gen.general_initial_condition(probs, nc0, 4)
    mueq = 1e-3 if nc + nct else 1e-8
    ex = [EXPONENTS[b % len(EXPONENTS)] for b in range(B)]
    scaled, mu_b = gen.scale_instances(probs, ex, mueq)
    c = 2.0 ** np.array(ex, dtype=np.float64)
    for prog in progs:
        base = run_cuda(gar, probs, dims, np.full(B, mueq), prog, kkt=True)
        got = run_cuda(gar, scaled, dims, mu_b, prog, kkt=True)
        assert np.all(base["status"] == 0) and np.all(got["status"] == 0), prog
        for k in EXACT + SCALED:
            want = base[k] * c.reshape((B,) + (1,) * (base[k].ndim - 1)) if k in SCALED else base[k]
            assert np.array_equal(got[k], want, equal_nan=True), (prog, k)
        assert np.array_equal(got["kkt"][:, 1:], base["kkt"][:, 1:] * c[:, None]), prog


# ---------------------------------------------------------------------------------------------------------------------
# kkt_error against exact residuals
# ---------------------------------------------------------------------------------------------------------------------
def exact_residual_rows(p, sol, mu):
    """lqrComputeKktError's residual rows evaluated exactly from the fp64 problem and solution: {family: [(r_i, T_i,
    m_i)]} with r_i the exact residual, T_i the sum of the magnitudes of its terms and m_i their number."""
    F = Fraction
    xs, us, vs, vsT, lbd0, lbdas = (sol[k] for k in ("xs", "us", "vs", "vsT", "lbd0", "lbdas"))
    N = p.horizon
    rows = {"dyn": [], "cst": [], "dual": []}

    def row(fam, terms):
        terms = [F(float(a)) * F(float(b)) for a, b in terms]
        rows[fam].append((sum(terms, F(0)), sum((abs(t) for t in terms), F(0)), len(terms)))

    nc0 = p.nc0
    for i in range(nc0):
        row("dyn", [(p.g0[i], 1.0)] + [(p.G0[i, c], xs[0][c]) for c in range(p.stages[0].nx)])
    for t, k in enumerate(p.stages):
        term = t == N
        x = xs[t]
        u = np.zeros(0) if term else us[t]
        v = vsT if term else vs[t]
        nx, nuu, ncc = k.nx, (0 if term else k.nu), len(v)
        for i in range(ncc):
            row("cst", [(k.d[i], 1.0), (-mu, v[i])] + [(k.C[i, c], x[c]) for c in range(nx)]
                + [(k.D[i, c], u[c]) for c in range(nuu)])
        lamn = None if term else lbdas[t]
        for i in range(nx):
            terms = [(k.q[i], 1.0)] + [(k.Q[i, c], x[c]) for c in range(nx)] + [(k.C[c, i], v[c]) for c in range(ncc)]
            terms += [(k.S[i, c], u[c]) for c in range(nuu)]
            terms += [(p.G0[c, i], lbd0[c]) for c in range(nc0)] if t == 0 else [(-1.0, lbdas[t - 1][i])]
            if not term:
                terms += [(k.A[c, i], lamn[c]) for c in range(nx)]
            row("dual", terms)
        for i in range(nuu):
            row("dual", [(k.r[i], 1.0)] + [(k.S[c, i], x[c]) for c in range(nx)] + [(k.D[c, i], v[c]) for c in range(ncc)]
                + [(k.R[i, c], u[c]) for c in range(k.nu)] + [(k.B[c, i], lamn[c]) for c in range(nx)])
        if not term:
            for i in range(nx):
                row("dyn", [(k.f[i], 1.0), (-1.0, xs[t + 1][i])] + [(k.A[i, c], x[c]) for c in range(nx)]
                    + [(k.B[i, c], u[c]) for c in range(k.nu)])
    return rows


def kkt_bounds(rows):
    """[lo, hi] for the fp64 infinity norm of each family: max_i(|r_i| -+ gamma_m T_i), gamma_m = m u / (1 - m u)."""
    u = Fraction(2) ** -53
    out = []
    for fam in ("dyn", "cst", "dual"):
        if not rows[fam]:
            out.append((0.0, 0.0))
            continue
        g = lambda m: (m + 1) * u / (1 - (m + 1) * u)
        lo = max(max(abs(r) - g(m) * T, Fraction(0)) for r, T, m in rows[fam])
        hi = max(abs(r) + g(m) * T for r, T, m in rows[fam])
        out.append((lo, hi))
    return out


@pytest.mark.parametrize("dims,nc0,per_instance_mu", [
    ((4, 2, 2, 2, 8), 0, False), ((4, 2, 2, 2, 8), 2, False), ((4, 2, 2, 2, 8), 4, False),
    ((12, 6, 0, 0, 8), 0, False), ((12, 6, 0, 0, 8), 6, False), ((12, 6, 0, 0, 8), 12, False),
    ((9, 5, 3, 2, 6), 4, False), ((4, 2, 2, 3, 8), 4, True), ((12, 6, 6, 2, 5), 12, True)])
def test_kkt_error_against_exact_residuals(gar, dims, nc0, per_instance_mu):
    """On solved problems (residuals ~1e-15, the regime where ab2_gar_kkt_error judges full-size batches): the device's
    infinity norms lie within the rounding bound of the exact residuals of the device's own solution."""
    nx, nu, nc, nct, N = dims
    B = 4
    probs = gen.generate_batch(81, B, N, nx, nu, nc, nct)
    if nc0 != nx:
        gen.general_initial_condition(probs, nc0, 5)
    mu = 1e-3 if nc + nct else 1e-8
    mueq = np.array([mu, 10 * mu, 0.1 * mu, mu])[:B] if per_instance_mu else mu
    got = run_cuda(gar, probs, dims, mueq, DEFAULT, kkt=True)
    assert np.all(got["status"] == 0)
    mus = np.broadcast_to(np.asarray(mueq, dtype=np.float64), (B,))
    for b, p in enumerate(probs):
        sol = {k: got[k][b] for k in ("xs", "us", "vs", "vsT", "lbd0", "lbdas")}
        for j, (lo, hi) in enumerate(kkt_bounds(exact_residual_rows(p, sol, mus[b]))):
            e = Fraction(float(got["kkt"][b, j]))
            assert lo <= e <= hi, (b, j, float(got["kkt"][b, j]), float(lo), float(hi))
        assert got["kkt"][b].max() <= 1e-9
