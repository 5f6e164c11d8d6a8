"""The adjoint of the LQ solve on the CPU: the numpy restatement (lq_adjoint_ref.py) of the adjoint problem and the
gradient records against central finite differences of the dense solve and against the dense adjoint -w z^T read
out of the KKT matrix's blocks; and the argument checks of aligator_b200.autograd.lq_solve."""
import numpy as np
import pytest

import gen
import lq_adjoint_ref as ref

MU = 1e-2
STAGE_BLOCKS = ("A", "B", "f", "Q", "S", "R", "q", "r", "C", "D", "d")
TERM_BLOCKS = ("Q", "q", "C", "d")

# (nx, nu, nc, nct, nc0, N)
CASES = [(3, 2, 1, 1, 3, 4), (3, 2, 0, 0, 1, 1), (4, 2, 1, 0, 0, 4), (4, 3, 0, 1, 4, 0), (5, 2, 1, 1, 1, 4),
         (5, 2, 0, 0, 5, 1), (4, 2, 1, 1, 0, 1), (3, 1, 1, 1, 1, 0), (5, 3, 1, 0, 0, 0), (4, 2, 0, 1, 1, 4)]
IDS = ["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d" % c for c in CASES]


def _problem(case, seed):
    nx, nu, nc, nct, nc0, N = case
    p = gen.generate_batch(seed, 1, N, nx, nu, nc, nct)
    return gen.general_initial_condition(p, nc0, seed)[0]


def _cotangent(case, seed):
    rng = np.random.default_rng(seed + 1000)
    return {k: rng.standard_normal(s) for k, s in ref._shapes(case[:6], 1).items()}


def _records(p, case):
    """Packed (padded) single-instance records of problem p."""
    nx, nu, nc, nct, nc0, N = case
    _, srec = ref.stage_offsets(nx, nu, nc)
    stage = np.zeros((1, N, srec))
    for t in range(N):
        r = gen.stage_record(p.stages[t])
        stage[0, t, :r.size] = r
    return (stage, gen.term_record(p.stages[N])[None], np.asarray(p.G0).ravel(order="F")[None],
            np.asarray(p.g0)[None])


def _dims(p):
    k0, kN = p.stages[0], p.stages[-1]
    N = p.horizon
    return (kN.nx, k0.nu if N else 0, k0.nc if N else 0, kN.nc, p.nc0, N)


def _solve(p):
    return ref.solution_dict([gen.lqr_dense_solve(p, MU)], _dims(p))


def _loss(p, cot):
    z = _solve(p)
    return sum(float(np.sum(cot[k] * z[k])) for k in ref.KEYS if z[k].size)


def _oracle_grads(p, case, cot):
    """The restatement: adjoint problem solved densely (as a problem of its own), then the gradient records."""
    z = _solve(p)
    st, tt, G0, g0 = ref.adjoint_records(*_records(p, case), cot, case)
    q = p.copy()
    nx, nu, nc, nct, nc0, N = case
    so, _ = ref.stage_offsets(nx, nu, nc)
    to, _ = ref.term_offsets(nx, nct)
    for t in range(N):
        for k in ("q", "r", "d", "f"):
            getattr(q.stages[t], k)[:] = st[0, t, so[k][0]:so[k][1]]
    for k in ("q", "d"):
        getattr(q.stages[N], k)[:] = tt[0, to[k][0]:to[k][1]]
    q.g0 = g0[0]
    w = _solve(q)
    return ref.grad_records(z, w, case)


def _block(rec, off, shape):
    a, b = off
    return rec[a:b].reshape(shape[1], shape[0]).T if len(shape) == 2 else rec[a:b]


def _families(p, case, g):
    """Gradient records -> {family: stacked array} over knots, in block form."""
    nx, nu, nc, nct, nc0, N = case
    so, _ = ref.stage_offsets(nx, nu, nc)
    to, _ = ref.term_offsets(nx, nct)
    fam = {}
    for t in range(N):
        k = p.stages[t]
        for n in STAGE_BLOCKS:
            fam.setdefault(n, []).append(_block(g["stage"][0, t], so[n], getattr(k, n).shape))
    kN = p.stages[N]
    for n in TERM_BLOCKS:
        fam["term_" + n] = [_block(g["term"][0], to[n], getattr(kN, n).shape)]
    fam["G0"] = [np.asarray(g["G0"][0]).reshape(nx, nc0).T]
    fam["g0"] = [g["g0"][0]]
    return {n: np.concatenate([np.ravel(a) for a in v]) for n, v in fam.items()}


def _finite_differences(p, case, cot, h=1e-6):
    nx, nu, nc, nct, nc0, N = case
    fam = {}

    def fd(arr, idx, sym):
        def bump(s):
            if sym and idx[0] != idx[1]:  # the symmetric argument: Q_ij and Q_ji together, as (P + P^T) / 2 does
                arr[idx] += s / 2
                arr[idx[::-1]] += s / 2
            else:
                arr[idx] += s
        bump(h)
        lp = _loss(p, cot)
        bump(-2 * h)
        lm = _loss(p, cot)
        bump(h)
        return (lp - lm) / (2 * h)

    def walk(name, arr, sym=False):
        out = np.zeros(arr.shape)
        for idx in np.ndindex(arr.shape):
            out[idx] = fd(arr, idx, sym)
        fam.setdefault(name, []).append(out)

    for t in range(N):
        k = p.stages[t]
        for n in STAGE_BLOCKS:
            walk(n, getattr(k, n), n in ("Q", "R"))
    kN = p.stages[N]
    for n in TERM_BLOCKS:
        walk("term_" + n, getattr(kN, n), n == "Q")
    p.G0 = np.array(p.G0, dtype=np.float64)
    p.g0 = np.array(p.g0, dtype=np.float64)
    walk("G0", p.G0)
    walk("g0", p.g0)
    return {n: np.concatenate([np.ravel(a) for a in v]) for n, v in fam.items()}


def _dense_adjoint(p, case, cot):
    """-w z^T of the whole KKT system, read out of its blocks (dh = -w)."""
    nx, nu, nc, nct, nc0, N = case
    K, rhs, offs = gen.lqr_dense_kkt(p, MU)
    z = np.linalg.solve(K, -rhs)
    zbar = np.zeros_like(z)
    zbar[:nc0] = cot["lam0"][0]
    for t in range(N + 1):
        o, m = offs[t], p.stages[t]
        zbar[o:o + nx] = cot["xs"][0, t]
        if t < N:
            zbar[o + nx:o + nx + nu] = cot["us"][0, t]
            zbar[o + nx + nu:o + nx + nu + nc] = cot["vs"][0, t]
            zbar[o + nx + nu + nc:o + 2 * nx + nu + nc] = cot["lams"][0, t]
        else:
            zbar[o + nx:o + nx + nct] = cot["vsT"][0]
    w = np.linalg.solve(K.T, zbar)
    G = -np.outer(w, z)
    two = lambda r, c, nr, ncol: G[r:r + nr, c:c + ncol] + G[c:c + ncol, r:r + nr].T
    sym = lambda r, n: 0.5 * (G[r:r + n, r:r + n] + G[r:r + n, r:r + n].T)
    fam = {}
    add = lambda n, a: fam.setdefault(n, []).append(np.ravel(a))
    for t in range(N):
        o = offs[t]
        ox, ou, oc, ol = o, o + nx, o + nx + nu, o + nx + nu + nc
        add("A", two(ol, ox, nx, nx))
        add("B", two(ol, ou, nx, nu))
        add("f", -w[ol:ol + nx])
        add("Q", sym(ox, nx))
        add("S", two(ox, ou, nx, nu))
        add("R", sym(ou, nu))
        add("q", -w[ox:ox + nx])
        add("r", -w[ou:ou + nu])
        add("C", two(oc, ox, nc, nx))
        add("D", two(oc, ou, nc, nu))
        add("d", -w[oc:oc + nc])
    o = offs[N]
    add("term_Q", sym(o, nx))
    add("term_q", -w[o:o + nx])
    add("term_C", two(o + nx, o, nct, nx))
    add("term_d", -w[o + nx:o + nx + nct])
    add("G0", two(0, nc0, nc0, nx))
    add("g0", -w[:nc0])
    return {n: np.concatenate(v) for n, v in fam.items()}


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_oracle_matches_finite_differences(case):
    seed = sum(c * 7 ** i for i, c in enumerate(case))
    p = _problem(case, seed)
    cot = _cotangent(case, seed)
    got = _families(p, case, _oracle_grads(p, case, cot))
    fd = _finite_differences(p, case, cot)
    assert set(got) == set(fd)
    for n in fd:
        if fd[n].size:
            assert gen.rel_fro(got[n], fd[n]) <= 1e-6, (n, gen.rel_fro(got[n], fd[n]))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_oracle_matches_dense_adjoint(case):
    seed = sum(c * 5 ** i for i, c in enumerate(case))
    p = _problem(case, seed)
    cot = _cotangent(case, seed)
    got = _families(p, case, _oracle_grads(p, case, cot))
    want = _dense_adjoint(p, case, cot)
    assert set(got) == set(want)
    for n in want:
        if want[n].size:
            assert gen.rel_fro(got[n], want[n]) <= 1e-12, (n, gen.rel_fro(got[n], want[n]))


def test_adjoint_records_keep_matrices_and_zero_pad():
    case = (4, 2, 1, 1, 4, 2)  # stage record of 69 doubles, padded to 70
    p = _problem(case, 3)
    recs = _records(p, case)
    st, tt, G0, g0 = ref.adjoint_records(*recs, {}, case)
    so, srec = ref.stage_offsets(4, 2, 1)
    assert srec == 70 and so["d"][1] == 69
    for n in ("A", "B", "Q", "S", "R", "C", "D"):
        assert np.array_equal(st[..., so[n][0]:so[n][1]], recs[0][..., so[n][0]:so[n][1]])
    for n in ("f", "q", "r", "d"):  # a missing cotangent is zero
        assert not np.any(st[..., so[n][0]:so[n][1]])
    assert np.array_equal(G0, recs[2]) and not np.any(g0)
    z = _solve(p)
    g = ref.grad_records(z, z, case)
    assert np.all(g["stage"][..., 69] == 0.0)


@pytest.fixture(scope="module")
def autograd():
    import __graft_entry__ as g
    g.build()
    import aligator_b200.autograd as ag
    return ag


def _unbuilt_handle(gar, nx, nu, nc, nct, nc0, N, B):
    """A CudaRiccatiBatch carrying the dimensions only (no device handle): enough for the argument checks, which
    run before any library call."""
    s = gar.CudaRiccatiBatch.__new__(gar.CudaRiccatiBatch)
    s.h = None
    s.dims = gar.GarDims(nx, nu, nc, nct, nc0, N, B, 0)
    s.srec, s.trec = gar.stage_record_doubles(nx, nu, nc), gar.term_record_doubles(nx, nct)
    return s


def test_lq_solve_rejects_cpu_float32_and_bad_shapes(autograd):
    import torch
    import aligator_b200.gar as gar
    nx, nu, nc, nct, nc0, N, B = 4, 2, 2, 1, 4, 3, 2
    s = _unbuilt_handle(gar, nx, nu, nc, nct, nc0, N, B)
    args = dict(stage=torch.zeros(B, N, s.srec, dtype=torch.float64), term=torch.zeros(B, s.trec, dtype=torch.float64),
                G0=torch.zeros(B, nc0 * nx, dtype=torch.float64), g0=torch.zeros(B, nc0, dtype=torch.float64))
    with pytest.raises(ValueError):  # CPU tensors
        autograd.lq_solve(s, mueq=1e-2, **args)
    for k in args:
        bad = dict(args)
        bad[k] = args[k].float()
        with pytest.raises(ValueError):
            autograd.lq_solve(s, mueq=1e-2, **bad)
    with pytest.raises(ValueError):
        autograd.lq_solve(object(), mueq=1e-2, **args)


def test_record_builders_match_the_packed_layout(autograd):
    import torch
    case = (3, 2, 1, 1, 3, 2)
    p = _problem(case, 5)
    stage, term, _, _ = _records(p, case)
    T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64))
    ks = p.stages
    blk = lambda n: torch.stack([T(getattr(ks[t], n)) for t in range(2)])[None]
    got = autograd.stage_records(*[blk(n) for n in STAGE_BLOCKS])
    assert np.array_equal(got.numpy(), stage)
    kN = ks[2]
    got_t = autograd.term_records(T(kN.Q)[None], T(kN.q)[None], T(kN.C)[None], T(kN.d)[None])
    assert np.array_equal(got_t.numpy(), term)
