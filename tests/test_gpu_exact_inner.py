"""The kernels that close the device-resident inner iteration, element by element against exact arithmetic
(tests/exact_inner_ref.py), and the FDDP backward pass against the extended-precision restatement (hp_reference).

Per output element: copies, zeroed rows, the normal-cone projection and every linear-step element bit for bit; every other
element within gamma_{m+1} T of its exact value.  FDDP: per family, e_kernel <= max(16 e_oracle, 64 u).  The Fraction
work runs on sampled instances: the first, the last, both sides of the grid-stride boundaries (8448 warps for the
per-instance kernels on 132 SMs; every cap of 1 to 8 CTAs per SM for the warp-per-record kernels) where the batch
reaches them, and both sides of per-instance value changes."""
import numpy as np
import pytest

import exact_inner_ref as xr
import gen
import hp_reference as hp
from exact_bounds import same_bits
from oracle import fddp as of
from inner_cases import fddp_args, fddp_case

pytestmark = pytest.mark.gpu

INF = np.inf
KINDS = 5  # equality, negative orthant, box [-0.5, 0.5], pinned box [0.25, 0.25], half-infinite box [-1, inf)


@pytest.fixture(scope="module")
def gar():
    import torch
    assert torch.cuda.is_available()
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    return gar


def T(a):
    import torch
    return torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device="cuda")


def cm(a):
    """math layout [.., rows, cols] -> the device's column-major blocks"""
    return np.ascontiguousarray(np.swapaxes(a, -1, -2))


def bounds(n, shift=0):
    k = (np.arange(n) + shift) % KINDS
    lo = np.select([k == 0, k == 1, k == 2, k == 3], [INF, -INF, -0.5, 0.25], -1.0)
    hi = np.select([k == 0, k == 1, k == 2, k == 3], [INF, 0.0, 0.5, 0.25], INF)
    return lo, hi


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def warp_cap():
    """Warps of the per-instance kernels' grid: 8 CTAs of 8 warps on every SM (8448 on 132 SMs).  Warp w serves
    instances w, w + cap, w + 2 cap, ..."""
    return 64 * sm_count()


def sample(B, *extra):
    """Instances checked against the host: first, last, both sides of the first and second grid-stride boundaries of
    the per-instance kernels, a few more."""
    W = warp_cap()
    s = {0, 1, B // 2, B - 2, B - 1, W - 1, W, W + 1, 2 * W - 1, 2 * W, *extra}
    return sorted(b for b in s if 0 <= b < B)


def record_boundaries(per_instance_records):
    """Instances holding the records on both sides of every grid-stride boundary a warp-per-record kernel can have:
    its grid is capped at p CTAs of 8 warps per SM, p = 1 .. 8 as its occupancy allows (the gradient kernel's 64 KB
    tile gives p = 3 on an H100), so records 8 p SMs - 1 and 8 p SMs (and twice that) end one pass and start the next."""
    out = set()
    for p in range(1, 9):
        W = 8 * p * sm_count()
        out.update(k // per_instance_records for k in (W - 1, W, 2 * W - 1, 2 * W))
    return out


def per_instance(B, base, seed):
    """[batch] values that change at every instance: base 2^((b mod 7) - 3) (1 + 0.1 (b mod 3))."""
    b = np.arange(B)
    return base * 2.0 ** ((b + seed) % 7 - 3) * (1 + 0.1 * (b % 3))


def expect_clean(where, fails):
    assert not fails, "%s: %d elements off, first %s" % (where, len(fails), fails[:3])


# ---------------------------------------------------------------------------------------------------------------------
# multipliers
# ---------------------------------------------------------------------------------------------------------------------
SHAPES = [  # N, nx, nu, nc, nct, nc0, B
    (10, 6, 3, 0, 0, 6, 7),      # C1 dims
    (8, 12, 6, 0, 0, 12, 5),     # C2 dims
    (6, 4, 2, 2, 2, 4, 33),      # C3 dims, terminal constraints
    (3, 57, 28, 0, 0, 57, 2),    # C5 dims
    (4, 2, 5, 3, 1, 1, 6),       # nu > nx
    (0, 4, 2, 0, 3, 4, 5),       # N = 0
    (1, 3, 2, 4, 0, 0, 5),       # N = 1, nc0 = 0
    (5, 4, 2, 0, 3, 2, 4),       # nc = 0, nct > 0, nc0 = nx / 2
    (3, 4, 2, 40, 35, 2, 4),     # nc, nct > 32
    (2, 3, 2, 3, 2, 3, 9000),    # past the grid-stride boundary
]


def mult_inputs(rng, N, nx, nc, nct, nc0, B, mu):
    r = lambda *s: rng.standard_normal(s)
    h = dict(xs=r(B, N + 1, nx), lam0=r(B, nc0), lams=r(B, N, nx), vs=r(B, N, nc), vsT=r(B, nct), prev_vs=r(B, N, nc),
             prev_vsT=r(B, nct), init_value=r(B, nc0), cval=r(B, N, nc), cval_N=r(B, nct), xnext=r(B, N, nx))
    lo, hi = bounds(nc)
    loN, hiN = bounds(nct, 1)
    # shifted exactly on lo / hi (prev = 0) and at -0.0 / +0.0, row by row, on the first knot and the terminal rows
    def edges(cval, prev, lo_, hi_, b):
        for i in range(cval.shape[-1]):
            e = (b + i) % 5
            if e == 0 and np.isfinite(lo_[i]):
                cval[i], prev[i] = lo_[i], 0.0
            elif e == 1 and np.isfinite(hi_[i]):
                cval[i], prev[i] = hi_[i], 0.0
            elif e == 2:
                cval[i], prev[i] = -0.0, -0.0
            elif e == 3:
                cval[i], prev[i] = 0.0, -0.0
    for b in range(min(B, 64)):
        if N and nc:
            edges(h["cval"][b, 0], h["prev_vs"][b, 0], lo, hi, b)
        edges(h["cval_N"][b], h["prev_vsT"][b], loN, hiN, b)
    h["fs"] = h["xnext"] - h["xs"][:, 1:]
    return h, (lo, hi, loN, hiN)


def run_multipliers(gar, s, h, bnd, mode, mu, mu_dyn):
    import torch
    B, N, nx = h["lams"].shape
    nc, nct, nc0 = h["vs"].shape[2], h["vsT"].shape[1], h["lam0"].shape[1]
    e = lambda *sh: torch.full(sh, float("nan"), device="cuda", dtype=torch.float64)
    out = dict(slack=e(B, N, nx), lam0_plus=e(B, nc0), lams_plus=e(B, N, nx), vs_plus=e(B, N, nc), vsT_plus=e(B, nct),
               shifted=e(B, N, nc), shifted_N=e(B, nct), Lv=e(B, N, nc), Lv_N=e(B, nct))
    keys = ["xs", "lam0", "lams", "vs", "vsT", "prev_vs", "prev_vsT", "init_value", "cval", "cval_N", mode]
    inp = {k: T(h[k]) for k in keys}
    inp.update({k: T(v) for k, v in zip(("lo", "hi", "loN", "hiN"), bnd)})
    sc = s.multipliers(inp, out, mu, mu_dyn)
    return {k: v.cpu().numpy() for k, v in out.items()}, sc


def check_multipliers(h, got, sc, bnd, mode, mus, mu_dyns, idx):
    lo, hi, loN, hiN = bnd
    for b in idx:
        one = {k: h[k][b] for k in h}
        if mode == "xnext":
            one["fs"] = None
        g = {k: v[b] for k, v in got.items()}
        assert sc[b, 1] == xr.flag(g) == 1.0, b
        w = xr.multipliers(one, g, lo, hi, loN, hiN, mus[b], mu_dyns[b])
        for k in ("slack", "lam0_plus", "lams_plus", "shifted", "shifted_N", "vs_plus", "vsT_plus", "Lv", "Lv_N"):
            expect_clean("%s instance %d" % (k, b), xr.failures(g[k], w[k]))
        # the projection on the device's own shifted, as the restatement-based test asserted it
        mu_inv = 1.0 / mus[b]
        N, nc = g["shifted"].shape
        nc_dev = np.array([[xr.normal_cone(g["shifted"][t, i], lo[i], hi[i]) for i in range(nc)] for t in range(N)])
        assert np.all(same_bits(g["vs_plus"], mu_inv * nc_dev.reshape(N, nc)))
        from fractions import Fraction
        assert w["prim"][0] <= Fraction(float(sc[b, 0])) <= w["prim"][1], (b, sc[b, 0], float(w["prim"][1]))


@pytest.mark.parametrize("mode", ["xnext", "fs"])
@pytest.mark.parametrize("pi", [False, True], ids=["scalar", "v"])
@pytest.mark.parametrize("shape", SHAPES, ids=[str(s) for s in SHAPES])
def test_multipliers_exact(gar, shape, pi, mode):
    N, nx, nu, nc, nct, nc0, B = shape
    rng = np.random.default_rng(sum(shape))
    mu, mu_dyn = 0.03, 0.007
    h, bnd = mult_inputs(rng, N, nx, nc, nct, nc0, B, mu)
    mus = per_instance(B, mu, 0) if pi else np.full(B, mu)
    mu_dyns = per_instance(B, mu_dyn, 3) if pi else np.full(B, mu_dyn)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    got, sc = run_multipliers(gar, s, h, bnd, mode, T(mus) if pi else mu, T(mu_dyns) if pi else mu_dyn)
    assert np.all(sc[:, 1] == 1.0)
    check_multipliers(h, got, sc, bnd, mode, mus, mu_dyns, sample(B))
    s.close()


FAMILIES = ("init_value", "lam0", "xnext", "xs", "lams", "cval", "prev_vs", "vs", "cval_N", "prev_vsT", "vsT")


@pytest.mark.parametrize("mode", ["xnext", "fs"])
@pytest.mark.parametrize("pi", [False, True], ids=["scalar", "v"])
def test_multipliers_flag_non_finite(gar, pi, mode):
    """NaN, +inf, -inf planted in one instance per input family; lams + f / mu_dyn overflowing from finite inputs;
    a non-finite xs[0] (which enters no output).  The flag is 0 exactly on the instances whose outputs are not finite
    and 1 on all others, and the untouched instances still meet their bounds."""
    N, nx, nu, nc, nct, nc0 = 3, 4, 2, 5, 3, 2
    fams = [f for f in FAMILIES if mode == "xnext" or f not in ("xnext", "xs")] + ([] if mode == "xnext" else ["fs"])
    B = 3 * len(fams) + 3 + 8
    rng = np.random.default_rng(7)
    mu, mu_dyn = 0.03, 0.007
    h, bnd = mult_inputs(rng, N, nx, nc, nct, nc0, B, mu)
    want = np.ones(B)
    b = 0
    for f in fams:
        for v in (np.nan, np.inf, -np.inf):
            a = h[f][b]
            if f == "xs":
                a[1 + b % N, b % nx] = v
            else:
                a.reshape(-1)[b % a.size] = v
            want[b] = 0.0
            b += 1
    h["fs"] = h["xnext"] - h["xs"][:, 1:] if mode == "xnext" else h["fs"]
    h["lams"][b, 1, 2] = 1.5e308                           # finite inputs, lams + f / mu_dyn overflows
    h["xnext"][b, 1, 2] = 1e307
    h["fs"][b, 1, 2] = 1e307
    want[b] = 0.0
    b += 1
    for v in (np.nan, np.inf):                              # xs[0] is no input of any output
        h["xs"][b, 0, 1] = v
        b += 1
    mus = per_instance(B, mu, 0) if pi else np.full(B, mu)
    mu_dyns = per_instance(B, mu_dyn, 3) if pi else np.full(B, mu_dyn)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    got, sc = run_multipliers(gar, s, h, bnd, mode, T(mus) if pi else mu, T(mu_dyns) if pi else mu_dyn)
    assert np.array_equal(sc[:, 1], want), np.nonzero(sc[:, 1] != want)
    assert all(xr.flag({k: v[i] for k, v in got.items()}) == want[i] for i in range(B))
    check_multipliers(h, got, sc, bnd, mode, mus, mu_dyns, [i for i in range(B) if want[i] == 1.0])
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# Lagrangian gradient and criterion
# ---------------------------------------------------------------------------------------------------------------------
GRAD_SHAPES = SHAPES[:-1] + [
    (2, 20, 14, 0, 0, 13, 3),    # rows 33: wmax 31, the first chunk straddles column nx = 20
    (3, 12, 6, 0, 0, 12, 3),     # rows 24: wmax 32, one chunk
    (2, 3, 2, 2, 1, 3, 9000),    # 27000 records, 9000 instances: past the gradient's and the criterion's grids
]


def grad_inputs(rng, N, nx, nu, nc, nct, nc0, B):
    r = lambda *s: rng.standard_normal(s)
    return dict(lx=r(B, N, nx), lu=r(B, N, nu), lx_N=r(B, nx), Jx=r(B, N, nx, nx), Ju=r(B, N, nx, nu),
                cJx=r(B, N, nc, nx), cJu=r(B, N, nc, nu), cJx_N=r(B, nct, nx), G0=r(B, nc0, nx), lam0=r(B, nc0),
                lams=r(B, N, nx), vs=r(B, N, nc), vsT=r(B, nct))


@pytest.mark.parametrize("shape", GRAD_SHAPES, ids=[str(s) for s in GRAD_SHAPES])
def test_lagrangian_gradient_and_criterion_exact(gar, shape):
    import torch
    N, nx, nu, nc, nct, nc0, B = shape
    rng = np.random.default_rng(sum(shape) + 1)
    g = grad_inputs(rng, N, nx, nu, nc, nct, nc0, B)
    mats = ("Jx", "Ju", "cJx", "cJu", "cJx_N", "G0")
    dev = {k: T(cm(v) if k in mats else v) for k, v in g.items()}
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    e = lambda *sh: torch.full(sh, float("nan"), device="cuda", dtype=torch.float64)
    idx = sample(B, *record_boundaries(N + 1))
    knots = None if N <= 12 else sorted({0, 1, N // 2, N - 1, N})
    for force in (False, True):
        o = dict(Lx=e(B, N, nx), Lx_N=e(B, nx), Lu=e(B, N, nu), Lxs=e(B, N + 1, nx), Lus=e(B, N, nu))
        s.lagrangian_gradient(dev, o, force_initial_condition=force)
        got = {k: v.cpu().numpy() for k, v in o.items()}
        assert np.all(same_bits(got["Lx"], got["Lxs"][:, :N])) and np.all(same_bits(got["Lx_N"], got["Lxs"][:, N]))
        assert np.all(same_bits(got["Lu"], got["Lus"]))
        for b in idx:
            wx, wu = xr.lagrangian_gradient({k: v[b] for k, v in g.items()}, force, knots)
            for t in (range(N + 1) if knots is None else knots):
                expect_clean("Lxs[%d] instance %d force %s" % (t, b, force), xr.failures(got["Lxs"][b, t], wx[t]))
                if t < N:
                    expect_clean("Lus[%d] instance %d" % (t, b), xr.failures(got["Lus"][b, t], wu[t]))
    # criterion: exact maxima of the device's arrays, every instance
    rng2 = np.random.default_rng(3)
    extra = dict(init_value=rng2.standard_normal((B, nc0)), slack=rng2.standard_normal((B, N, nx)),
                 Lv=rng2.standard_normal((B, N, nc)), Lv_N=rng2.standard_normal((B, nct)))
    arrs = dict(Lxs=o["Lxs"], Lus=o["Lus"], **{k: T(v) for k, v in extra.items()})
    ch = s.criterion(arrs)
    cd = e(B, 2)
    s.criterion(arrs, out=cd)
    assert np.all(same_bits(cd.cpu().numpy(), ch))
    for b in range(B):
        assert tuple(ch[b]) == xr.criterion(got["Lxs"][b], got["Lus"][b], extra["init_value"][b], extra["slack"][b],
                                             extra["Lv"][b], extra["Lv_N"][b]), b
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# assembly
# ---------------------------------------------------------------------------------------------------------------------
ASM_SHAPES = [  # N, nx, nu, nc, nct, nc0, B, Hessians, Hxx0
    (4, 6, 3, 0, 0, 6, 7, True, True),
    (3, 12, 6, 0, 0, 12, 5, True, False),
    (5, 4, 2, 2, 2, 4, 33, False, True),
    (2, 57, 28, 0, 0, 57, 2, True, True),
    (3, 2, 5, 3, 1, 1, 6, True, True),
    (0, 4, 2, 0, 3, 4, 5, False, True),
    (1, 3, 2, 4, 0, 0, 5, True, False),
    (4, 4, 2, 0, 3, 2, 4, False, False),
    (2, 4, 2, 40, 35, 2, 4, True, True),
    (1, 3, 2, 3, 2, 3, 9000, True, True),   # 9000 stage records and 9000 terminal knots, nct > 0
]


def asm_inputs(rng, N, nx, nu, nc, nct, nc0, B, hess, h0):
    r = lambda *s: rng.standard_normal(s)
    inp = dict(Jx=r(B, N, nx, nx), Ju=r(B, N, nx, nu), slack=r(B, N, nx), Lxx=r(B, N, nx, nx), Lxu=r(B, N, nx, nu),
               Luu=r(B, N, nu, nu), Lx=r(B, N, nx), Lu=r(B, N, nu), Lxx_N=r(B, nx, nx), Lx_N=r(B, nx),
               cJx=r(B, N, nc, nx), cJu=r(B, N, nc, nu), Lv=r(B, N, nc), shifted=r(B, N, nc),
               cJx_N=r(B, nct, nx), Lv_N=r(B, nct), shifted_N=r(B, nct), G0=r(B, nc0, nx), g0=r(B, nc0))
    if hess:
        inp.update(Hxx=0.01 * r(B, N, nx, nx), Hxu=0.01 * r(B, N, nx, nu), Huu=0.01 * r(B, N, nu, nu))
    if h0:
        inp["Hxx0"] = 0.01 * r(B, nx, nx)
    lo, hi = bounds(nc)
    loN, hiN = bounds(nct, 2)
    for b in range(min(B, 64)):   # shifted on the bounds (inactive), at +-0, just outside
        for sh, lo_, hi_ in ([(inp["shifted"][b, t], lo, hi) for t in range(N)] + [(inp["shifted_N"][b], loN, hiN)]):
            for i in range(sh.size):
                e = (b + i) % 7
                if e == 0 and np.isfinite(lo_[i]):
                    sh[i] = lo_[i]
                elif e == 1 and np.isfinite(hi_[i]):
                    sh[i] = hi_[i]
                elif e == 2:
                    sh[i] = -0.0
                elif e == 3:
                    sh[i] = 0.0
                elif e == 4 and np.isfinite(hi_[i]):
                    sh[i] = np.nextafter(hi_[i], INF)
    inp.update(lo=lo, hi=hi, loN=loN, hiN=hiN)
    return inp


@pytest.mark.parametrize("pi", [False, True], ids=["scalar", "v"])
@pytest.mark.parametrize("shape", ASM_SHAPES, ids=[str(s) for s in ASM_SHAPES])
def test_assemble_exact(gar, shape, pi):
    N, nx, nu, nc, nct, nc0, B, hess, h0 = shape
    rng = np.random.default_rng(sum(shape[:7]))
    inp = asm_inputs(rng, N, nx, nu, nc, nct, nc0, B, hess, h0)
    pregs = per_instance(B, 1e-3, 1) if pi else np.full(B, 1.5e-3)
    mu_invs = per_instance(B, 1e3, 2) if pi else np.full(B, 1e3)
    shared = ("lo", "hi", "loN", "hiN")
    mats = ("Jx", "Ju", "Lxx", "Lxu", "Luu", "Hxx", "Hxu", "Huu", "cJx", "cJu", "Lxx_N", "cJx_N", "G0", "Hxx0")
    dev = {k: T(cm(v) if k in mats else v) for k, v in inp.items()}
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    s.assemble(dev, T(pregs) if pi else pregs[0], T(mu_invs) if pi else mu_invs[0])
    s.synchronize()
    srec, trec = gar.stage_record_doubles(nx, nu, nc), gar.term_record_doubles(nx, nct)
    stage = s.get_problem(0).reshape(B, N, srec)
    term = s.get_problem(1).reshape(B, trec)
    G0 = s.get_problem(2).reshape(B, nc0 * nx)
    g0 = s.get_problem(3).reshape(B, nc0)
    for b in sample(B, *record_boundaries(max(N, 1))):
        one = {k: (v if k in shared else v[b]) for k, v in inp.items()}
        w = xr.assemble(one, N, nx, nu, nc, nct, nc0, pregs[b], mu_invs[b])
        for t in range(N):
            blk = xr.stage_blocks(stage[b, t], nx, nu, nc)
            for n in xr.STAGE_ORDER:
                expect_clean("stage %s t %d instance %d" % (n, t, b), xr.failures(blk[n], w["stages"][t][n]))
            assert np.all(same_bits(blk["pad"], 0.0)), (b, t)
        blk = xr.term_blocks(term[b], nx, nct)
        for n in ("Q", "q", "C", "d"):
            expect_clean("term %s instance %d" % (n, b), xr.failures(blk[n], w["term"][n]))
        assert np.all(same_bits(G0[b], cm(w["G0"]).ravel())) and np.all(same_bits(g0[b], w["g0"]))
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# line search
# ---------------------------------------------------------------------------------------------------------------------
LS_SHAPES = [  # nx, nu, nc, nct, N, B
    (6, 3, 0, 0, 10, 7), (12, 6, 0, 0, 8, 5), (4, 2, 2, 3, 6, 33), (12, 6, 6, 2, 5, 4), (3, 2, 0, 0, 3, 9000),
]


def swept(gar, nx, nu, nc, nct, N, B, seed):
    """A handle whose outputs hold the step of a solved problem (a few generated problems tiled over the batch)."""
    nb = min(B, 8)
    probs = gen.generate_batch(seed, nb, N, nx, nu, nc, nct)
    packed = gar.pack_problems(probs)
    reps = -(-B // nb)
    packed = [np.concatenate([a.reshape(nb, -1)] * reps)[:B] for a in packed]
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B)
    s.set_problem(*packed)
    s.sweep(1e-3 if nc + nct else 1e-8)
    assert np.all(s.status() == 0)
    step = {k: s.get(w) for k, w in dict(xs=gar.OUT_XS, us=gar.OUT_US, vs=gar.OUT_VS, vsT=gar.OUT_VST,
                                         lam0=gar.OUT_LBD0, lams=gar.OUT_LBDAS).items()}
    return s, step


@pytest.mark.parametrize("shape", LS_SHAPES, ids=[str(s) for s in LS_SHAPES])
def test_linear_step_bit_exact(gar, shape):
    import torch
    nx, nu, nc, nct, N, B = shape
    s, step = swept(gar, nx, nu, nc, nct, N, B, 21)
    rng = np.random.default_rng(sum(shape))
    cur_h = {k: rng.standard_normal(v.shape) for k, v in step.items()}
    alphas = per_instance(B, 0.37, 0)
    for pi in (False, True):
        alpha = T(alphas) if pi else 0.37
        a = alphas if pi else np.full(B, 0.37)
        cur = {k: T(v) for k, v in cur_h.items()}
        trial = {k: torch.full_like(v, float("nan")) for k, v in cur.items()}
        s.linear_step(alpha, cur, trial)
        out = {k: v.cpu().numpy() for k, v in trial.items()}
        s.linear_step(alpha, cur, cur)                      # in place (trial is current), as the refinement calls it
        inplace = {k: v.cpu().numpy() for k, v in cur.items()}
        for b in sample(B):
            for k in cur_h:
                want = xr.linear_step(cur_h[k][b], step[k][b], a[b])
                assert np.all(same_bits(out[k][b], want)), (pi, k, b)
                assert np.all(same_bits(inplace[k][b], want)), (pi, k, b, "in place")
    s.close()


def cancelling(L, d, rng, offset):
    """Rewrite L so that the products L_i d_i cancel exactly in pairs across the flattened (x, u) arrays -- pairs that
    straddle x and u and different knots: L_p = 2^s d_q, L_q = -2^s d_p, so L_p d_p + L_q d_q = 0 in exact arithmetic,
    with s in [-4, 4] varying the pairs' sizes.  With ``offset`` != 0, one entry then moves the exact sum to about
    ``offset`` times sum |L d|."""
    n = L.size
    perm = rng.permutation(n)
    for p, q in zip(perm[0::2], perm[1::2]):
        sc = 2.0 ** int(rng.integers(-4, 5))
        L[p], L[q] = sc * d[q], -sc * d[p]
    if n % 2:
        L[perm[-1]] = 0.0
    if offset:
        k = perm[0]
        L[k] += offset * float(np.sum(np.abs(L * d))) / d[k]
    return L


@pytest.mark.parametrize("case", ["random", "cancel0", "cancel1e-12", "long"])
def test_directional_derivative_and_al_value_exact(gar, case):
    import torch
    nx, nu, nc, nct, N, B = (3, 2, 0, 0, 1000, 4) if case == "long" else (3, 2, 0, 2, 3, 9000)
    if case == "long":
        assert (N + 1) * nx % 64 != 0   # the second accumulation chain ends unevenly
    s, step = swept(gar, nx, nu, nc, nct, N, B, 5)
    rng = np.random.default_rng(9)
    Lxs, Lus = rng.standard_normal((B, N + 1, nx)), rng.standard_normal((B, N, nu))
    idx = sample(B)
    if case != "random":
        for b in idx:
            L = np.concatenate([Lxs[b].ravel(), Lus[b].ravel()])
            d = np.concatenate([step["xs"][b].ravel(), step["us"][b].ravel()])
            L = cancelling(L, d, rng, 1e-12 if case == "cancel1e-12" else 0.0)
            Lxs[b], Lus[b] = L[:Lxs[b].size].reshape(N + 1, nx), L[Lxs[b].size:].reshape(N, nu)
    d1 = s.directional_derivative(T(Lxs), T(Lus))
    for b in idx:
        w = xr.directional_derivative(Lxs[b], Lus[b], step["xs"][b], step["us"][b])
        if case in ("cancel0", "long"):
            assert w.exact == 0 and w.T > 0
        elif case != "random":
            assert 0.5e-12 * w.T <= abs(w.exact) <= 2e-12 * w.T
        expect_clean("directional derivative %d" % b, xr.failures(np.array([d1[b]]), np.array([w], dtype=object)))
    # the AL value: NULL cost or a cost, nct = 0 and > 0, scalar and per-instance penalties
    plus = dict(lam0=rng.standard_normal((B, nx)), lams=rng.standard_normal((B, N, nx)),
                vs=rng.standard_normal((B, N, nc)), vsT=rng.standard_normal((B, nct)))
    cost = rng.standard_normal(B)
    pd = {k: T(v) for k, v in plus.items()}
    for pi in (False, True):
        mudyn = per_instance(B, 0.01, 0) if pi else np.full(B, 0.01)
        mucstr = per_instance(B, 7.0, 4) if pi else np.full(B, 7.0)
        for c in (None, cost):
            val = s.al_value(pd, None if c is None else T(c), T(mudyn) if pi else 0.01, T(mucstr) if pi else 7.0)
            for b in idx:
                w = xr.al_value(None if c is None else c[b], plus["lam0"][b], plus["lams"][b], plus["vs"][b],
                                plus["vsT"][b], mudyn[b], mucstr[b])
                expect_clean("al_value %d" % b, xr.failures(np.array([val[b]]), np.array([w], dtype=object)))
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# FDDP backward pass at the conditioning bar
# ---------------------------------------------------------------------------------------------------------------------
FDDP_CASES = [  # name, nx, nu, N, B
    ("plain", 12, 6, 30, 9), ("plain", 6, 3, 20, 5), ("plain", 14, 7, 25, 4), ("plain", 9, 4, 10, 3),
    ("singular", 6, 3, 12, 4), ("defects", 12, 6, 10, 4), ("plain", 4, 2, 1, 6),
    ("plain", 3, 2, 3, 9000),
]


@pytest.mark.parametrize("pi", [False, True], ids=["scalar", "v"])
@pytest.mark.parametrize("case", FDDP_CASES, ids=["%s-%d-%d-%d-%d" % c for c in FDDP_CASES])
def test_fddp_backward_pass_at_the_bar(gar, case, pi):
    import torch
    name, nx, nu, N, B = case
    rng = np.random.default_rng(nx + N)
    d, preg = fddp_case(name, rng, B, N, nx, nu)
    pregs = preg * (1 + 0.5 * (np.arange(B) % 3)) if pi else np.full(B, preg)
    vec = ("fs", "Lx", "Lu", "Lx_N")
    arr = {k: T(v if k in vec else cm(v)) for k, v in d.items()}
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    Vx = torch.empty(B, N + 1, nx, dtype=torch.float64, device="cuda")
    Qk = torch.empty(B, N, nu, dtype=torch.float64, device="cuda")
    s.fddp_backward_pass(arr, T(pregs) if pi else preg, Vx, Qk)
    s.synchronize()
    assert np.all(s.status() == 0)
    fb, ff, V = s.get(gar.OUT_FB), s.get(gar.OUT_FF), s.get(gar.OUT_VXX)
    Vx, Qk = Vx.cpu().numpy(), Qk.cpu().numpy()
    idx = sample(B) if B > 16 else list(range(min(B, 4)))
    got, orc, ref = [], [], []
    for b in idx:
        args = fddp_args(d, b)
        ref.append(hp.fddp_backward_pass(*args, pregs[b]))
        orc.append(of.backward_pass(*args, pregs[b]))
        got.append(dict(K=list(fb[b, :, :nu]), k=list(ff[b, :, :nu]), Vxx=list(V[b]), Vx=list(Vx[b]), Quuks=list(Qk[b])))
    e_o, e_k = hp.fddp_errors(orc, ref), hp.fddp_errors(got, ref)
    print("\n" + hp.table("fddp %s nx %d nu %d N %d B %d%s" % (name, nx, nu, N, B, " (per-instance preg)" if pi else ""),
                          e_o, e_k))
    assert not hp.violations(e_k, e_o), hp.violations(e_k, e_o)
    s.close()
