"""GPU parity tests: the CUDA path, called through the C ABI, against the CPU oracle on
identical inputs.  Bar (BASELINE.json north_star): K, k, Vxx within 1e-10 relative
Frobenius of the reference algorithm; KKT residuals within the reference's own test
thresholds (tests/gar/riccati.cpp).  Every launch variant is exercised."""
import numpy as np
import pytest

import gen
from oracle import gar_oracle as orc

pytestmark = pytest.mark.gpu

TOL = 1e-10  # fp64 relative Frobenius, north_star


@pytest.fixture(scope="module")
def gar():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    return gar


def run_cuda(gar, probs, nx, nu, nc, nct, N, mueq, variant=-1, split_calls=False):
    stage, term, G0, g0 = gar.pack_problems(probs)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, probs[0].nc0, N, len(probs), 0, variant)
    s.set_problem(stage, term, G0, g0)
    if split_calls:
        s.backward(mueq)
        s.forward()
    else:
        s.sweep(mueq)
    out = {k: s.get(w) for k, w in dict(
        ff=gar.OUT_FF, fb=gar.OUT_FB, Vxx=gar.OUT_VXX, vx=gar.OUT_VX, ffT=gar.OUT_FFT,
        fbT=gar.OUT_FBT, xs=gar.OUT_XS, us=gar.OUT_US, vs=gar.OUT_VS, vsT=gar.OUT_VST,
        lbd0=gar.OUT_LBD0, lbdas=gar.OUT_LBDAS).items()}
    out["status"] = s.status()
    out["launches"] = s.launch_count()
    s.close()
    return out, (stage, term, G0, g0)


def compare(got, ref, nu, nc, N, mueq, tol=TOL):
    assert np.all(got["status"] == 0)
    worst = {}

    def upd(k, a, b):
        worst[k] = max(worst.get(k, 0.0), gen.rel_fro(a, b))

    B = ref["xs"].shape[0]
    for b in range(B):
        for t in range(N):
            upd("K", got["fb"][b, t, :nu], ref["fb"][b, t, :nu])
            upd("k", got["ff"][b, t, :nu], ref["ff"][b, t, :nu])
            upd("fb", got["fb"][b, t], ref["fb"][b, t])
            upd("ff", got["ff"][b, t], ref["ff"][b, t])
        for t in range(N + 1):
            upd("Vxx", got["Vxx"][b, t], ref["Vxx"][b, t])
            upd("vx", got["vx"][b, t], ref["vx"][b, t])
        for key in ("xs", "us", "vs", "lbdas", "lbd0", "vsT", "ffT", "fbT"):
            if ref[key].size:
                upd(key, got[key][b], ref[key][b])
    # K on control-constrained knots is bounded by eps*cond(KKT) ~ 6e-17/mueq between any two
    # correct fp64 solvers (SURVEY Appendix C); everything else is gated at tol.
    tolk = max(tol, 2.4e-16 / mueq) if nc > 0 else tol
    bad = {k: v for k, v in worst.items() if not v <= (tolk if k in ("K", "k") else tol)}
    assert not bad, (bad, worst)
    return worst


def oracle_batch(probs, packed, nx, nu, nc, nct, N, mueq):
    bo = orc.BatchedOracle(nx, nu, nc, nct, probs[0].nc0, N, len(probs), *packed)
    bo.sweep(mueq)
    assert np.all(bo.status == 1)
    return bo.get()


SHAPES = [  # (nx, nu, nc, nct, N, batch, mueq)
    (6, 3, 0, 0, 100, 5, 1e-8),      # BASELINE config 1 dims
    (12, 6, 0, 0, 100, 37, 1e-11),   # config 2 dims (bench mueq), ragged batch
    (4, 2, 2, 0, 100, 67, 1e-3),     # config 3 dims, gated mueq
    (4, 2, 2, 0, 100, 33, 1e-6),     # config 3 dims, gated mueq
    (14, 7, 0, 0, 200, 9, 1e-8),     # config 4 dims
    (2, 2, 0, 0, 16, 11, 1e-14),
    (2, 2, 2, 0, 8, 13, 1e-4),
    (3, 2, 0, 0, 50, 10, 1e-8),
    (5, 2, 2, 0, 20, 7, 1e-3),
    (8, 3, 0, 0, 30, 6, 1e-8),
    (10, 4, 0, 0, 100, 3, 1e-12),
    (12, 6, 6, 0, 20, 5, 1e-3),      # NK = 12 > 8: cooperative shared-memory BK
    (4, 2, 0, 0, 25, 130, 1e-8),
]


@pytest.mark.parametrize("shape", SHAPES)
def test_cuda_matches_oracle(gar, shape):
    nx, nu, nc, nct, N, B, mueq = shape
    probs = gen.generate_batch(100 + nx, B, N, nx, nu, nc, nct)
    got, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq)
    ref = oracle_batch(probs, packed, nx, nu, nc, nct, N, mueq)
    compare(got, ref, nu, nc, N, mueq)
    assert got["launches"] == 1  # one persistent launch per sweep


@pytest.mark.parametrize("variant", [0, 1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("shape", [(12, 6, 0, 0, 40, 19, 1e-8), (4, 2, 2, 0, 40, 70, 1e-3),
                                   (6, 3, 0, 0, 30, 9, 1e-8)])
def test_all_launch_variants(gar, shape, variant):
    nx, nu, nc, nct, N, B, mueq = shape
    probs = gen.generate_batch(7, B, N, nx, nu, nc, nct)
    got, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq, variant=variant)
    ref = oracle_batch(probs, packed, nx, nu, nc, nct, N, mueq)
    compare(got, ref, nu, nc, N, mueq)


def test_backward_then_forward_equals_fused_sweep(gar):
    nx, nu, nc, nct, N, B, mueq = 12, 6, 0, 0, 30, 8, 1e-8
    probs = gen.generate_batch(3, B, N, nx, nu, nc, nct)
    a, _ = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq, split_calls=False)
    b, _ = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq, split_calls=True)
    for k in ("fb", "ff", "Vxx", "xs", "us", "lbdas"):
        assert np.array_equal(a[k], b[k]), k
    assert b["launches"] == 2


def test_terminal_constraints_and_edge_horizons(gar):
    for (nx, nu, nc, nct, N, B, mueq) in [(4, 2, 2, 3, 12, 5, 1e-3), (6, 3, 0, 2, 10, 4, 1e-2),
                                         (4, 2, 0, 0, 0, 3, 1e-8), (4, 2, 0, 0, 1, 3, 1e-8)]:
        probs = gen.generate_batch(11, B, N, nx, nu, nc, nct)
        got, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq)
        ref = oracle_batch(probs, packed, nx, nu, nc, nct, N, mueq)
        compare(got, ref, nu, nc, N, mueq)


def test_reference_style_generator_reaches_reference_kkt_thresholds(gar):
    """A ~ U[-1,1], singular Q (tests/gar/test_util.cpp style): KKT residual of the CUDA
    solution within the reference's thresholds (tests/gar/riccati.cpp:84,138)."""
    from aligator_b200.lqr import lqr_initialize_solution
    nx, nu, N = 6, 3, 100
    rng = np.random.default_rng(5)
    prob = gen.generate_lq_problem(rng, rng.standard_normal(nx), N, nx, nu, 0, 0, True)
    solver = gar.ProximalRiccatiSolver(prob)
    mueq = 1e-12
    assert solver.backward(mueq)
    xs, us, vs, lbdas = lqr_initialize_solution(prob)
    assert solver.forward(xs, us, vs, lbdas)
    op = orc.OracleProblem(prob)
    osol = orc.OracleSolution(op)
    osol.set(xs, us, vs, lbdas)
    assert max(orc.kkt_error(op, osol, mueq)) <= 1e-9
    # and the gains are the oracle's
    ref = orc.ProximalRiccatiSolver(op)
    ref.backward(mueq)
    for t in (0, N // 2, N - 1):
        f = ref.factor(t)
        assert gen.rel_fro(solver.getFeedback(t), f["fb"]) <= TOL
        assert gen.rel_fro(solver.getFeedforward(t), f["ff"]) <= TOL


def test_riccati_short_horz_pb_on_gpu(gar):
    """tests/gar/riccati.cpp:26-85 on the CUDA path: the one constrained knot of the
    reference test is expressed by padding every knot to nc=2 with zero rows (inactive
    rows give z = 0 exactly; documented in INTEGRATION.md)."""
    from aligator_b200.lqr import LqrKnot, LqrProblem, lqr_initialize_solution
    mueq = 1e-8
    rng = np.random.default_rng(4)
    nx = nu = 2
    horz = 8
    Brnd, frnd = rng.uniform(-1, 1, (nx, nu)), rng.uniform(-1, 1, nx)

    def init_knot(nu_, nc):
        k = LqrKnot(nx, nu_, nc)
        k.A[:] = [[0.1, 0.0], [-0.1, 0.01]]
        if nu_:
            k.B[:] = Brnd
            k.R[:] = 0.1 * np.eye(nu_)
        k.f[:] = frnd
        k.Q[:] = 0.01 * np.eye(nx)
        return k

    knots = [init_knot(nu, 2) for _ in range(horz)]
    knots[4].D[:] = np.eye(nu)
    knots[4].d[:] = 0.1
    term = init_knot(0, 0)
    term.Q[:] = np.eye(nx)
    term.q[:] = np.ones(nx)
    prob = LqrProblem(knots + [term], nx)
    prob.g0[:] = -np.ones(nx)
    prob.G0[:] = np.eye(nx)
    solver = gar.ProximalRiccatiSolver(prob)
    solver.backward(mueq)
    xs, us, vs, lbdas = lqr_initialize_solution(prob)
    solver.forward(xs, us, vs, lbdas)
    op = orc.OracleProblem(prob)
    osol = orc.OracleSolution(op)
    osol.set(xs, us, vs, lbdas)
    assert max(orc.kkt_error(op, osol, mueq)) <= 1e-9


def test_singular_instance_is_flagged_not_thrown(gar):
    """R = 0, B = 0 on one instance: the reference throws 'Failed stage LDL
    factorization'; the batched path flags that instance and finishes the others."""
    nx, nu, N, B = 4, 2, 6, 4
    probs = gen.generate_batch(2, B, N, nx, nu, 0, 0)
    k = probs[2].stages[3]
    k.R[:] = 0.0
    k.B[:] = 0.0
    k.S[:] = 0.0
    stage, term, G0, g0 = gar.pack_problems(probs)
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    s.set_problem(stage, term, G0, g0)
    s.sweep(1e-8)
    st = s.status()
    assert st[2] & 1 and not st[0] and not st[1] and not st[3]
    with pytest.raises(gar.GarError):
        gar.ProximalRiccatiSolver(probs).backward(1e-8)


def test_device_resident_problem_and_outputs(gar):
    """Zero-copy path: problem buffers and result reads stay on the device (torch only
    provides the memory)."""
    import torch
    nx, nu, N, B = 12, 6, 20, 16
    probs = gen.generate_batch(9, B, N, nx, nu, 0, 0)
    stage, term, G0, g0 = gar.pack_problems(probs)
    dev = [torch.from_numpy(a).cuda() for a in (stage, term, G0, g0)]
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    st = torch.cuda.current_stream().cuda_stream
    s.set_problem(*dev, memspace=gar.AB2_DEVICE, stream=st)
    s.sweep(1e-8, stream=st)
    K0 = torch.empty(B, nu + nx, nx, dtype=torch.float64, device="cuda")
    s.get_range_into(gar.OUT_FB, 0, B, 0, 1, K0, gar.AB2_DEVICE, stream=st)
    torch.cuda.synchronize()
    ref = oracle_batch(probs, (stage, term, G0, g0), nx, nu, 0, 0, N, 1e-8)
    assert gen.rel_fro(K0.cpu().numpy(), ref["fb"][:, 0]) <= TOL


def test_cycle_append(gar):
    """cycleAppend (proximal-riccati.hxx:79-86): factors rotate left, slot N-1 is zeroed;
    after the caller rotates its problem a fresh backward matches the oracle."""
    nx, nu, N, B = 6, 3, 8, 3
    probs = gen.generate_batch(21, B, N, nx, nu, 0, 0)
    solver = gar.ProximalRiccatiSolver(probs)
    solver.backward(1e-8)
    before = [solver.getFeedback(t, 1).copy() for t in range(N)]
    rng = np.random.default_rng(0)
    new = [gen.generate_knot(rng, nx, nu, 0, conditioned=True) for _ in range(B)]
    solver.cycleAppend(new)
    for t in range(N - 1):
        assert np.array_equal(solver.getFeedback(t, 1), before[t + 1])
    assert np.all(solver.getFeedback(N - 1, 1) == 0)
    for p, k in zip(probs, new):  # what cycleProblem does to the problem
        p.stages = p.stages[1:N] + [k] + [p.stages[N]]
    solver.backward(1e-8)
    packed = gar.pack_problems(probs)
    ref = oracle_batch(probs, packed, nx, nu, 0, 0, N, 1e-8)
    for t in (0, N - 1):
        assert gen.rel_fro(solver.getFeedback(t, 2), ref["fb"][2, t]) <= TOL


def test_cycle_append_is_a_ring_shift(gar):
    """O(1) cycle_append: three cycles in a row WITHOUT re-uploading the problem.  The getters (whole arrays,
    sub-ranges, gains layout, the solver-owned problem) return knot order through the ring heads; a sweep on
    the cycled device copy equals the oracle on the rotated problem; the next backward resets the factor head."""
    nx, nu, N, B = 6, 3, 9, 4
    mueq = 1e-8
    probs = gen.generate_batch(33, B, N, nx, nu, 0, 0)
    stage, term, G0, g0 = gar.pack_problems(probs)
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    s.set_problem(stage, term, G0, g0)
    s.sweep(mueq)
    fb0, ff0, V0, vx0 = (s.get(w).copy() for w in (gar.OUT_FB, gar.OUT_FF, gar.OUT_VXX, gar.OUT_VX))
    gains0 = s.get_gains().copy()
    rng = np.random.default_rng(1)
    cur = [list(p.stages) for p in probs]
    for cyc in range(1, 4):
        new = [gen.generate_knot(rng, nx, nu, 0, conditioned=True) for _ in range(B)]
        s.cycle_append(np.stack([gar.pack_stage_knot(k, s.srec) for k in new]))
        fb, ff, V, vx = (s.get(w) for w in (gar.OUT_FB, gar.OUT_FF, gar.OUT_VXX, gar.OUT_VX))
        # factors: rotated left `cyc` times, the last `cyc` stage slots zero, the terminal entry in place
        assert np.array_equal(fb[:, :N - cyc], fb0[:, cyc:]) and np.all(fb[:, N - cyc:] == 0)
        assert np.array_equal(ff[:, :N - cyc], ff0[:, cyc:]) and np.all(ff[:, N - cyc:] == 0)
        assert np.array_equal(V[:, :N - cyc], V0[:, cyc:N]) and np.all(V[:, N - cyc:N] == 0) and np.array_equal(V[:, N], V0[:, N])
        assert np.array_equal(vx[:, N], vx0[:, N])
        # sub-range straddling the wrap point
        buf = np.empty(2 * 4 * (nu + nx) * nx)
        s.get_range_into(gar.OUT_FB, 1, 2, N - cyc - 3, 4, buf, gar.AB2_HOST)
        s.synchronize()
        assert np.array_equal(buf.reshape(2, 4, nu + nx, nx), fb[1:3, N - cyc - 3:N - cyc + 1])
        for p, c, k in zip(probs, cur, new):
            c[:] = c[1:N] + [k] + [c[N]]
        # the solver-owned problem in knot order
        st2 = s.get_problem(0).reshape(B, N, -1)
        for b in range(B):
            for t in (0, N - cyc, N - 1):
                assert np.array_equal(st2[b, t], gar.pack_stage_knot(cur[b][t], s.srec))
    # sweep straight from the cycled device copy (no set_problem): equals the oracle on the rotated problems
    s.sweep(mueq)
    from aligator_b200.lqr import LqrProblem
    rot = []
    for p, c in zip(probs, cur):
        q = p.copy()
        q.stages = c
        rot.append(q)
    packed = gar.pack_problems(rot)
    ref = oracle_batch(rot, packed, nx, nu, 0, 0, N, mueq)
    for key, what in (("fb", gar.OUT_FB), ("Vxx", gar.OUT_VXX), ("xs", gar.OUT_XS), ("lbdas", gar.OUT_LBDAS)):
        assert gen.rel_fro(s.get(what), ref[key]) <= TOL, key
    assert s.kkt_error(mueq).max() <= 1e-9
    s.close()


def test_full_size_properties_config2(gar):
    """BASELINE config 2 at full size (nx12 nu6 N100 batch4096): size-independent
    properties -- KKT residual of sampled instances within the reference thresholds,
    closed-loop consistency x_{t+1} = a_t + Ahat_t x_t, symmetry of Vxx_t (t>=1)."""
    nx, nu, N, B, mueq = 12, 6, 100, 4096, 1e-11
    rng = np.random.default_rng(0)
    base = gen.generate_batch(77, 16, N, nx, nu, 0, 0)
    stage16, term16, G016, g016 = gar.pack_problems(base)
    reps = B // 16
    scale = (1.0 + 0.01 * rng.standard_normal((reps, 1, 1, 1)))
    stage = (stage16[None] * scale).reshape(B, N, -1)
    term = np.tile(term16, (reps, 1))
    G0 = np.tile(G016, (reps, 1))
    g0 = np.tile(g016, (reps, 1))
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    s.set_problem(stage, term, G0, g0)
    s.sweep(mueq)
    assert np.all(s.status() == 0)
    X, U = s.get(gar.OUT_XS), s.get(gar.OUT_US)
    FB, FF, V = s.get(gar.OUT_FB), s.get(gar.OUT_FF), s.get(gar.OUT_VXX)
    xn = FF[:, :, nu:] + np.einsum("btij,btj->bti", FB[:, :, nu:], X[:, :-1])
    assert gen.rel_fro(xn, X[:, 1:]) <= 1e-12
    un = FF[:, :, :nu] + np.einsum("btij,btj->bti", FB[:, :, :nu], X[:, :-1])
    assert gen.rel_fro(un, U) <= 1e-12
    assert np.array_equal(V[:, 1:], V[:, 1:].transpose(0, 1, 3, 2))
    # sampled instances against the oracle
    idx = [0, 1, 17, 2048, 4095]
    bo = orc.BatchedOracle(nx, nu, 0, 0, nx, N, len(idx), stage[idx], term[idx], G0[idx], g0[idx])
    bo.sweep(mueq)
    ref = bo.get()
    assert gen.rel_fro(FB[idx], ref["fb"]) <= TOL and gen.rel_fro(V[idx], ref["Vxx"]) <= TOL
    assert gen.rel_fro(X[idx], ref["xs"]) <= TOL


@pytest.mark.parametrize("variant", [0, 1, 7])
@pytest.mark.parametrize("shape", [(6, 3, 0, 0, 12, 9), (12, 6, 0, 0, 30, 17), (2, 2, 0, 0, 6, 5)])
def test_unconstrained_knots_that_need_interchanges(gar, shape, variant):
    """nc = 0 but Rhat needs Bunch-Kaufman interchanges: the branch-free register fast
    path must detect it and fall back to the general algorithm."""
    nx, nu, nc, nct, N, B = shape
    probs = gen.make_pivoting(gen.generate_batch(31, B, N, nx, nu, nc, nct))
    got, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, 1e-8, variant=variant)
    ref = oracle_batch(probs, packed, nx, nu, nc, nct, N, 1e-8)
    compare(got, ref, nu, nc, N, 1e-8)


@pytest.mark.parametrize("variant", [7, 8, 10])
@pytest.mark.parametrize("shape", [(12, 6, 0, 0, 100, 41, 1e-11), (14, 7, 0, 0, 200, 9, 1e-8),
                                   (10, 4, 0, 0, 50, 7, 1e-8), (12, 6, 0, 2, 10, 5, 1e-2)])
def test_tensor_core_variants(gar, shape, variant):
    """Variants 7/8/10: the stage step on the FP64 tensor cores (DMMA m8n8k4); 10 = single
    record buffer."""
    nx, nu, nc, nct, N, B, mueq = shape
    probs = gen.generate_batch(55 + nx, B, N, nx, nu, nc, nct)
    got, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq, variant=variant)
    ref = oracle_batch(probs, packed, nx, nu, nc, nct, N, mueq)
    compare(got, ref, nu, nc, N, mueq)


BLOCK_SHAPES = [  # (nx, nu, nc, nct, N, batch, mueq): no compile-time instantiation -> CTA per instance
    (7, 3, 0, 0, 30, 9, 1e-8),
    (9, 5, 3, 0, 20, 7, 1e-3),
    (20, 9, 0, 0, 40, 5, 1e-8),
    (13, 4, 0, 2, 12, 300, 1e-2),     # more instances than resident CTAs: the persistent loop
    (24, 20, 20, 0, 6, 3, 1e-3),      # 40 KKT rows, 48 rows in the initial-stage system
    (57, 28, 0, 0, 25, 4, 1e-8),      # BASELINE config 5 dims (Talos whole-body)
    (1, 1, 0, 0, 5, 3, 1e-8),
]


@pytest.mark.parametrize("shape", BLOCK_SHAPES)
def test_block_kernel_runtime_shapes(gar, shape):
    """Shapes without a compile-time instantiation run the CTA-per-instance kernel
    (riccati_block.cuh): DMMA-tiled products over the CTA's warps, thread-per-row BK."""
    nx, nu, nc, nct, N, B, mueq = shape
    assert gar.supported(nx, nu, nc, nx) == 2
    probs = gen.generate_batch(200 + nx, B, N, nx, nu, nc, nct)
    got, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq)
    ref = oracle_batch(probs, packed, nx, nu, nc, nct, N, mueq)
    compare(got, ref, nu, nc, N, mueq)
    assert got["launches"] == 1


@pytest.mark.parametrize("shape", [(12, 6, 0, 0, 40, 19, 1e-8), (4, 2, 2, 0, 40, 70, 1e-3),
                                   (12, 6, 6, 0, 20, 5, 1e-3)])
def test_block_kernel_forced_on_instantiated_shapes(gar, shape):
    """variant 9 forces the CTA-per-instance kernel; same results as the oracle, and the
    split backward()/forward() calls reproduce the fused sweep bit for bit."""
    nx, nu, nc, nct, N, B, mueq = shape
    probs = gen.generate_batch(9, B, N, nx, nu, nc, nct)
    got, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq, variant=9)
    ref = oracle_batch(probs, packed, nx, nu, nc, nct, N, mueq)
    compare(got, ref, nu, nc, N, mueq)
    got2, _ = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq, variant=9, split_calls=True)
    for k in ("fb", "ff", "Vxx", "xs", "us", "lbdas"):
        assert np.array_equal(got[k], got2[k]), k


def test_block_kernel_interchanges(gar):
    nx, nu, nc, nct, N, B = 9, 5, 0, 0, 12, 6
    probs = gen.make_pivoting(gen.generate_batch(31, B, N, nx, nu, nc, nct))
    got, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, 1e-8)
    ref = oracle_batch(probs, packed, nx, nu, nc, nct, N, 1e-8)
    compare(got, ref, nu, nc, N, 1e-8)


def test_shape_too_large_for_one_cta_is_refused(gar):
    assert gar.supported(120, 40, 0, 120) == 0
    with pytest.raises(gar.GarError):
        gar.CudaRiccatiBatch(120, 40, 0, 0, 120, 4, 2)


@pytest.mark.parametrize("shape,chunks", [((12, 6, 0, 0, 20, 37, 1e-8), 5), ((4, 2, 2, 3, 10, 64, 1e-3), 0),
                                          ((9, 5, 3, 0, 6, 11, 1e-3), 3), ((12, 6, 0, 0, 8, 3, 1e-8), 16)])
def test_pipelined_host_sweep_equals_plain_calls(gar, shape, chunks):
    """ab2_gar_sweep_host (upload / sweep / download pipelined over batch slices on internal
    streams) returns bit for bit what set_problem + sweep + get return."""
    import torch
    nx, nu, nc, nct, N, B, mueq = shape
    probs = gen.generate_batch(5, B, N, nx, nu, nc, nct)
    plain, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, probs[0].nc0, N, B)
    pin = [torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in packed]
    whats = dict(fb=gar.OUT_FB, ff=gar.OUT_FF, xs=gar.OUT_XS, us=gar.OUT_US, lbdas=gar.OUT_LBDAS,
                 Vxx=gar.OUT_VXX, vsT=gar.OUT_VST)
    outs = {w: torch.full((max(int(np.prod(s.out_shape(w))), 1),), np.nan, dtype=torch.float64).pin_memory()
            for w in whats.values()}
    for _ in range(2):  # twice: the internal streams/events are reused
        s.sweep_host(pin[0], pin[1], pin[2], pin[3], mueq, outs, nchunks=chunks)
        s.synchronize()
    for k, w in whats.items():
        got = outs[w].numpy()[:int(np.prod(s.out_shape(w)))].reshape(s.out_shape(w))
        if k == "Vxx":
            got = got.transpose(0, 1, 3, 2)
        assert np.array_equal(got, plain[k]), k
    assert np.all(s.status() == 0)
    # the results also stay on the device: a plain get sees them
    assert np.array_equal(s.get(gar.OUT_XS), plain["xs"])
    s.close()


@pytest.mark.parametrize("shape,chunks", [((12, 6, 0, 0, 9, 11, 1e-8), 3), ((4, 2, 2, 2, 7, 9, 1e-3), 2),
                                          ((9, 5, 3, 0, 5, 6, 1e-2), 0)])
def test_host_sweep_with_triangle_packed_records(gar, shape, chunks):
    """ab2_gar_sweep_host_sym: Q and R of every stage knot cross PCIe as lower triangles
    (ab2_gar_pack_stage_sym) and are rebuilt in HBM -- bit for bit the results of the plain host sweep
    (the generator's Q, R are exactly symmetric: wishart products)."""
    import torch
    nx, nu, nc, nct, N, B, mueq = shape
    probs = gen.generate_batch(8, B, N, nx, nu, nc, nct)
    for p in probs:  # exact symmetry, whatever the generator's arithmetic did
        for k in p.stages:
            k.Q[:] = 0.5 * (k.Q + k.Q.T)
            k.R[:] = 0.5 * (k.R + k.R.T)
    plain, packed = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, probs[0].nc0, N, B)
    sym = s.pack_stage_sym(np.ascontiguousarray(packed[0]))
    nsym = int(gar.lib().ab2_gar_stage_record_doubles_sym(nx, nu, nc))
    assert sym.size == B * N * nsym and nsym < s.srec
    pin = [torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in (sym,) + tuple(packed[1:])]
    whats = dict(fb=gar.OUT_FB, ff=gar.OUT_FF, xs=gar.OUT_XS, us=gar.OUT_US, lbdas=gar.OUT_LBDAS, Vxx=gar.OUT_VXX)
    outs = {w: torch.full((max(int(np.prod(s.out_shape(w))), 1),), np.nan, dtype=torch.float64).pin_memory()
            for w in whats.values()}
    for _ in range(2):
        s.sweep_host_sym(pin[0], pin[1], pin[2], pin[3], mueq, outs, nchunks=chunks)
        s.synchronize()
    for k, w in whats.items():
        got = outs[w].numpy()[:int(np.prod(s.out_shape(w)))].reshape(s.out_shape(w))
        if k == "Vxx":
            got = got.transpose(0, 1, 3, 2)
        assert np.array_equal(got, plain[k]), k
    assert np.all(s.status() == 0)
    s.close()


def test_first_step_policy_kernel(gar):
    """ab2_gar_first_step_policy packs [K_0 | k_0] exactly as the host-side reference packing
    of knot 0 of OUT_FB / OUT_FF (aligator_b200.sharding.pack_first_step_policy)."""
    import torch
    from aligator_b200 import sharding
    nx, nu, nc, nct, N, B, mueq = 12, 6, 0, 0, 10, 9, 1e-8
    probs = gen.generate_batch(3, B, N, nx, nu, nc, nct)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B)
    s.set_problem(*gar.pack_problems(probs))
    s.sweep(mueq)
    pol = torch.full((B, nu, nx + 1), float("nan"), dtype=torch.float64, device="cuda")
    s.first_step_policy_into(pol)
    s.synchronize()
    fb, ff = s.get(gar.OUT_FB), s.get(gar.OUT_FF)
    want = sharding.pack_first_step_policy(torch, torch.from_numpy(fb[:, 0]), torch.from_numpy(ff[:, 0]), nu, nx)
    assert torch.equal(pol.cpu(), want)
    s.close()


def test_gains_in_results_layout(gar):
    """ab2_gar_get_gains: column-major (nu+nc+nx) x (nx+1) blocks with column 0 = ff, the layout of
    results_.gains_ (solver-proxddp.hxx:619-626)."""
    nx, nu, nc, nct, N, B, mueq = 4, 2, 2, 0, 7, 5, 1e-3
    probs = gen.generate_batch(8, B, N, nx, nu, nc, nct)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B)
    s.set_problem(*gar.pack_problems(probs))
    s.sweep(mueq)
    g = s.get_gains()
    fb, ff = s.get(gar.OUT_FB), s.get(gar.OUT_FF)
    assert np.array_equal(g[:, :, 0, :], ff)
    assert np.array_equal(g[:, :, 1:, :], fb.transpose(0, 1, 3, 2))
    s.close()


def test_cuda_matches_committed_fixture(gar):
    """The CUDA path against the committed (oracle-generated) fixture tests/golden/oracle_regression.npz
    -- no oracle code runs in this test."""
    import importlib.util
    import os
    here = os.path.dirname(os.path.abspath(__file__))
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(here, "golden", "make_golden.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    ref = np.load(os.path.join(here, "golden", "oracle_regression.npz"))
    for case, (nx, nu, nc, nct, N, mueq, seed) in mg.CASES.items():
        probs = gen.generate_batch(seed, 2, N, nx, nu, nc, nct)
        got, _ = run_cuda(gar, probs, nx, nu, nc, nct, N, mueq)
        tol = TOL
        for k in ("fb", "ff", "Vxx", "vx", "xs", "us", "lbdas"):
            assert gen.rel_fro(got[k], ref["%s/%s" % (case, k)]) <= tol, (case, k)


@pytest.mark.parametrize("shape", [(12, 6, 0, 0, 20, 9, 1e-8), (4, 2, 2, 3, 12, 17, 1e-3), (9, 5, 3, 0, 6, 5, 1e-3)])
def test_kkt_error_kernel_matches_oracle(gar, shape):
    """ab2_gar_kkt_error (lqrComputeKktError on the device, gar/utils.hxx:88-182) against the oracle's
    restatement evaluated on the SAME solution, instance by instance: (a) on the solved problem the
    residuals are rounding noise (both below 1e-9, the reference's own test threshold is 1e-8/1e-9);
    (b) on a PERTURBED problem (same solution) they are O(1e-3) and must agree to 1e-9 relative."""
    nx, nu, nc, nct, N, B, mueq = shape
    probs = gen.generate_batch(21, B, N, nx, nu, nc, nct)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, probs[0].nc0, N, B)
    s.set_problem(*gar.pack_problems(probs))
    s.sweep(mueq)
    got = s.kkt_error(mueq)
    assert got.shape == (B, 3) and got.max() <= 1e-9, got.max()
    xs, us, vs, vsT = s.get(gar.OUT_XS), s.get(gar.OUT_US), s.get(gar.OUT_VS), s.get(gar.OUT_VST)
    lb, lb0 = s.get(gar.OUT_LBDAS), s.get(gar.OUT_LBD0)
    # perturb every block of the problem; the solution on the device stays that of the original
    rng = np.random.default_rng(5)
    for p in probs:
        for k in p.stages:
            for name in ("A", "B", "f", "Q", "S", "R", "q", "r", "C", "D", "d"):
                a = getattr(k, name)
                a[...] = a + 1e-3 * rng.standard_normal(a.shape)
        p.G0[...] = p.G0 + 1e-3 * rng.standard_normal(p.G0.shape)
        p.g0[...] = p.g0 + 1e-3 * rng.standard_normal(p.g0.shape)
    s.set_problem(*gar.pack_problems(probs))
    got = s.kkt_error(mueq)
    for b in range(B):
        op = orc.OracleProblem(probs[b])
        sol = orc.OracleSolution(op)
        sol.set(xs=[xs[b, t] for t in range(N + 1)], us=[us[b, t] for t in range(N)],
                vs=[vs[b, t] for t in range(N)] + [vsT[b]], lbdas=[lb0[b]] + [lb[b, t] for t in range(N)])
        ref = np.array(orc.kkt_error(op, sol, mueq))
        assert ref[0] > 1e-6 and ref[2] > 1e-6 and (ref[1] > 1e-6 or nc + nct == 0)  # the perturbation shows
        assert np.allclose(got[b], ref, rtol=1e-9, atol=0.0), (b, got[b], ref)
    s.close()


def test_kkt_error_of_every_instance_at_full_size(gar):
    """BASELINE config 2 at full size: the KKT residuals of ALL 4096 instances, computed on the device."""
    import torch
    sys_path_bench = __import__("bench")
    nx, nu, N, B = 12, 6, 100, 4096
    stage, term, G0, g0 = sys_path_bench.synth_batch_torch(torch, B, N, nx, nu, torch.device("cuda:0"), 7, 0)
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
    s.sweep(1e-11)
    assert np.all(s.status() == 0)
    e = s.kkt_error(1e-11)
    assert e.shape == (B, 3) and np.all(np.isfinite(e))
    assert e.max() <= 1e-8, e.max()
    s.close()


@pytest.mark.parametrize("shape", [(5, 2, 0, 0, 3, 6, 1e-8), (4, 3, 2, 0, 2, 5, 1e-3), (7, 3, 0, 2, 7, 4, 1e-2)])
def test_parametric_problems(gar, shape):
    """nth > 0 (riccati-kernel.hxx:185-192, 278-311; proximal-riccati.hxx:50-59; forward with theta)
    through the Python mirror of ProximalRiccatiSolver, against the oracle."""
    import lq_cases
    nx, nu, nc, nct, nth, N, mueq = shape
    probs = [lq_cases.make_problem(50 + b, N, nx, nu, nc, nct, nth) for b in range(3)]
    solver = gar.ProximalRiccatiSolver(probs)
    assert solver.backward(mueq)
    thetas = np.random.default_rng(1).standard_normal((3, nth))
    sols = [gar.lqr_initialize_solution(p) for p in probs] if hasattr(gar, "lqr_initialize_solution") else None
    tol = TOL
    for b, p in enumerate(probs):
        op = orc.OracleProblem(p)
        ref = orc.ProximalRiccatiSolver(op)
        assert ref.backward(mueq)
        for t in range(N):
            f = ref.factor(t)
            assert gen.rel_fro(solver.getFeedback(t, b), f["fb"]) <= tol
            assert gen.rel_fro(solver.getFeedbackTheta(t, b), f["fth"]) <= tol
        k0 = ref.kkt0()
        mine = solver.kkt0(b)
        for key in ("ff", "fth", "thGrad", "thHess"):
            assert gen.rel_fro(mine[key], k0[key]) <= tol, key
        for t in range(N + 1):
            f = ref.factor(t)
            assert gen.rel_fro(solver._get(gar.OUT_VXT)[b, t], f["Vxt"]) <= tol
            assert gen.rel_fro(solver._get(gar.OUT_VTT)[b, t], f["Vtt"]) <= tol
            assert gen.rel_fro(solver._get(gar.OUT_VT)[b, t], f["vt"]) <= tol
    # forward with theta
    solver.batch.forward(theta=thetas)
    X, U = solver.batch.get(gar.OUT_XS), solver.batch.get(gar.OUT_US)
    L0, L = solver.batch.get(gar.OUT_LBD0), solver.batch.get(gar.OUT_LBDAS)
    for b, p in enumerate(probs):
        op = orc.OracleProblem(p)
        ref = orc.ProximalRiccatiSolver(op)
        ref.backward(mueq)
        sol = orc.OracleSolution(op)
        assert ref.forward(sol, thetas[b])
        xs, us, vs, lb = sol.get()
        assert gen.rel_fro(X[b], np.array(xs)) <= tol and gen.rel_fro(U[b], np.array(us[:N])) <= tol
        assert gen.rel_fro(L0[b], lb[0]) <= tol and gen.rel_fro(L[b], np.array(lb[1:])) <= tol


@pytest.mark.parametrize("shape", [(4, 2, 0, 5, 1e-8), (6, 3, 2, 7, 1e-3), (12, 6, 0, 20, 1e-9), (5, 3, 2, 0, 1e-2)])
def test_terminal_knot_with_controls(gar, shape):
    """A terminal knot with nu > 0 (terminalSolve's second branch, riccati-kernel.hxx:150-173; the
    reference's lqr_initialize_solution then has N+1 controls, gar/utils.hpp:120-131) through the Python
    mirror: solved as one more stage knot before a null terminal knot; against the oracle, which
    restates the reference's branch directly."""
    nx, nu, nc, N, mueq = shape
    probs = []
    for b in range(3):
        rng = np.random.default_rng(900 + b)
        p = gen.generate_lq_problem(rng, rng.standard_normal(nx), N, nx, nu, nc=nc, singular=False, conditioned=True)
        p.stages[N] = gen.generate_knot(rng, nx, nu, nc, 0, False, conditioned=True)
        probs.append(p)
    solver = gar.ProximalRiccatiSolver(probs)
    assert solver.backward(mueq)
    sols = [gar.lqr_initialize_solution(p) for p in probs]
    assert all(len(s[1]) == N + 1 for s in sols)
    assert solver.forward(*[list(z) for z in zip(*sols)])
    for b, p in enumerate(probs):
        op = orc.OracleProblem(p)
        ref = orc.ProximalRiccatiSolver(op)
        assert ref.backward(mueq)
        for t in range(N + 1):
            f = ref.factor(t)
            rows = nu + nc if t == N else nu + nc + nx  # the terminal knot's co-state rows are never written
            assert gen.rel_fro(solver.getFeedback(t, b)[:rows], f["fb"][:rows]) <= TOL, t
            assert gen.rel_fro(solver.getFeedforward(t, b)[:rows], f["ff"][:rows]) <= TOL, t
            assert gen.rel_fro(solver.Vxx(t, b), f["Vxx"]) <= TOL and gen.rel_fro(solver.vx(t, b), f["vx"]) <= TOL
        assert np.all(solver.getFeedback(N, b)[nu + nc:] == 0.0)
        sol = orc.OracleSolution(op)
        assert ref.forward(sol)
        xs, us, vs, lb = sol.get()
        mx, mu_, mv, ml = sols[b]
        assert len(us) == N + 1
        for mine, theirs in ((mx, xs), (mu_, us), (mv, vs), (ml, lb)):
            assert gen.rel_fro(np.concatenate(mine), np.concatenate(theirs)) <= TOL


def test_ragged_stage_dims_and_terminal_controls(gar):
    """Every knot with its own (nu, nc) (gar/lqr-problem.hpp:49-118) AND a terminal knot with controls,
    through the Python mirror (padding to the largest dims, gar._pad_knot): factors, value functions and
    the solution against the oracle on the caller's unpadded problem."""
    from aligator_b200.lqr import LqrProblem
    nx, mueq = 6, 1e-4
    dims = [(3, 0), (2, 2), (3, 1), (1, 0), (3, 2), (2, 0), (2, 1)]  # the last one is the terminal knot
    N = len(dims) - 1
    probs = []
    for b in range(3):
        rng = np.random.default_rng(40 + b)
        knots = [gen.generate_knot(rng, nx, nu, nc, 0, False, conditioned=True) for nu, nc in dims]
        p = LqrProblem(knots, nx)
        p.G0[:] = -np.eye(nx)
        p.g0[:] = rng.standard_normal(nx)
        probs.append(p)
    solver = gar.ProximalRiccatiSolver(probs)
    assert solver.backward(mueq)
    sols = [gar.lqr_initialize_solution(p) for p in probs]
    assert solver.forward(*[list(z) for z in zip(*sols)])
    for b, p in enumerate(probs):
        op = orc.OracleProblem(p)
        ref = orc.ProximalRiccatiSolver(op)
        assert ref.backward(mueq)
        for t, (nu, nc) in enumerate(dims):
            f = ref.factor(t)
            rows = nu + nc if t == N else nu + nc + nx
            assert solver.getFeedback(t, b).shape[0] == nu + nc + nx
            assert gen.rel_fro(solver.getFeedback(t, b)[:rows], f["fb"][:rows]) <= TOL, t
            assert gen.rel_fro(solver.getFeedforward(t, b)[:rows], f["ff"][:rows]) <= TOL, t
            assert gen.rel_fro(solver.Vxx(t, b), f["Vxx"]) <= TOL and gen.rel_fro(solver.vx(t, b), f["vx"]) <= TOL
        sol = orc.OracleSolution(op)
        assert ref.forward(sol)
        for mine, theirs in zip(sols[b], sol.get()):
            assert [len(m) for m in mine] == [len(r) for r in theirs]
            assert gen.rel_fro(np.concatenate(mine), np.concatenate(theirs)) <= TOL


PAR_SHAPES = [  # (nx, nu, nc, nct, N, legs, batch, mueq)
    (4, 2, 0, 0, 11, 3, 3, 1e-8), (6, 3, 0, 0, 20, 4, 5, 1e-8), (4, 2, 2, 0, 13, 2, 4, 1e-3),
    (14, 7, 0, 0, 200, 8, 6, 1e-9),   # BASELINE config 4 dims, 8 legs of 25 knots
    (12, 6, 0, 0, 100, 6, 40, 1e-9),  # config 2 dims, the reference bench's thread count (bench/gar-riccati.cpp:87-90)
    (5, 3, 2, 2, 9, 3, 3, 1e-2), (7, 3, 0, 0, 7, 8, 2, 1e-8),
]


@pytest.mark.parametrize("shape", PAR_SHAPES)
def test_parallel_solver_on_device(gar, shape):
    """gar::ParallelRiccatiSolver on the device (ab2_gar_create_parallel): legs of ALL instances in one
    launch, condensed block-tridiagonal solve + refinement per instance in a second, legs' rollouts
    in a third.  Against the oracle's parallel solver (same leg split): every per-knot factor incl. the
    parametric ones at 1e-10, the rollout at 1e-9; against the serial solution at the reference's own
    thresholds (tests/gar/parallel.cpp:211-243: 1e-7) and through the KKT residuals of every instance."""
    nx, nu, nc, nct, N, T, B, mueq = shape
    probs = gen.generate_batch(90 + nx, B, N, nx, nu, nc, nct)
    stage, term, G0, g0 = gar.pack_problems(probs)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B, legs=T)
    s.set_problem(stage, term, G0, g0)
    s.backward(mueq)
    s.forward()
    assert np.all(s.status() == 0)
    assert s.launch_count() == 3
    out = {k: s.get(w) for k, w in dict(ff=gar.OUT_FF, fb=gar.OUT_FB, Vxx=gar.OUT_VXX, vx=gar.OUT_VX, fth=gar.OUT_FTH,
                                        Vxt=gar.OUT_VXT, Vtt=gar.OUT_VTT, vt=gar.OUT_VT, xs=gar.OUT_XS, us=gar.OUT_US,
                                        vs=gar.OUT_VS, lbd0=gar.OUT_LBD0, lbdas=gar.OUT_LBDAS).items()}
    kk = s.kkt_error(mueq)
    assert kk.max() <= 1e-7, kk.max()   # tests/gar/parallel.cpp:211,221
    for b in sorted({0, B // 2, B - 1}):
        op = orc.OracleProblem(probs[b].copy())
        par = orc.ParallelRiccatiSolver(op, T, threaded=False)
        assert par.backward(mueq)
        sol = orc.OracleSolution(op)
        par.forward(sol)
        for t in range(N):
            f = par.factor(t)
            assert gen.rel_fro(out["fb"][b, t], f["fb"]) <= TOL, ("fb", t)
            assert gen.rel_fro(out["ff"][b, t], f["ff"]) <= TOL, ("ff", t)
            if f["dims"][4]:
                assert gen.rel_fro(out["fth"][b, t], f["fth"]) <= TOL, ("fth", t)
        for t in range(N + 1):
            f = par.factor(t)
            assert gen.rel_fro(out["Vxx"][b, t], f["Vxx"]) <= TOL and gen.rel_fro(out["vx"][b, t], f["vx"]) <= TOL
            if f["dims"][4]:
                assert gen.rel_fro(out["Vxt"][b, t], f["Vxt"]) <= TOL, ("Vxt", t)
                assert gen.rel_fro(out["Vtt"][b, t], f["Vtt"]) <= TOL, ("Vtt", t)
                assert gen.rel_fro(out["vt"][b, t], f["vt"]) <= TOL
        xs, us, vs, lb = sol.get()
        assert gen.rel_fro(out["xs"][b], np.stack(xs)) <= 1e-9
        assert gen.rel_fro(out["us"][b], np.stack(us[:N])) <= 1e-9
        assert gen.rel_fro(out["lbdas"][b], np.stack(lb[1:])) <= 1e-9
        ops = orc.OracleProblem(probs[b])
        ser = orc.ProximalRiccatiSolver(ops)
        ser.backward(mueq)
        sols = orc.OracleSolution(ops)
        ser.forward(sols)
        xs2, us2, vs2, lb2 = sols.get()
        assert gen.rel_fro(out["xs"][b], np.stack(xs2)) <= 1e-7
        assert gen.rel_fro(out["lbdas"][b], np.stack(lb2[1:])) <= 1e-7
    # collapseFeedback as the reference states it (parallel-solver.hpp:41-51)
    s.collapse_feedback()
    fb0 = s.get(gar.OUT_FB)[0, 0, :nu]
    op = orc.OracleProblem(probs[0].copy())
    par = orc.ParallelRiccatiSolver(op, T, threaded=False)
    par.backward(mueq)
    par.collapseFeedback()
    assert gen.rel_fro(fb0, par.factor(0)["fb"][:nu]) <= TOL
    # the fused call and the pipelined host call take the same three launches per (sub-)batch
    s.sweep(mueq)
    assert np.array_equal(s.get(gar.OUT_XS), out["xs"])
    s.close()


def test_parallel_solver_python_mirror_and_errors(gar):
    """The Python mirror of the class (same constructor / call sequence as the reference) and its error
    behaviour: num_threads < 2 raises (parallel-solver.hxx:42-46)."""
    nx, nu, N = 6, 3, 20
    p = gen.generate_batch(5, 1, N, nx, nu, 0, 0)[0]
    with pytest.raises(gar.GarError):
        gar.ParallelRiccatiSolver(p, 1)
    solver = gar.ParallelRiccatiSolver(p, 4)
    assert solver.getNumThreads() == 4
    assert solver.backward(1e-9)
    xs = [np.zeros(nx) for _ in range(N + 1)]
    us = [np.zeros(nu) for _ in range(N)]
    vs = [np.zeros(0) for _ in range(N + 1)]
    lb = [np.zeros(nx) for _ in range(N + 1)]
    assert solver.forward(xs, us, vs, lb)
    ops = orc.OracleProblem(p)
    ser = orc.ProximalRiccatiSolver(ops)
    ser.backward(1e-9)
    sol = orc.OracleSolution(ops)
    ser.forward(sol)
    xs2, us2, _, lb2 = sol.get()
    assert gen.rel_fro(np.stack(xs), np.stack(xs2)) <= 1e-8 and gen.rel_fro(np.stack(us), np.stack(us2)) <= 1e-8
    assert gen.rel_fro(np.stack(lb), np.stack(lb2)) <= 1e-8
    solver.collapseFeedback()
    assert solver.getFeedback(0).shape == (nu + nx, nx)


def test_peer_memory_policy_allgather_two_gpus(gar):
    """Fused pack + NVLink peer-memory all-gather (ab2_gar_policy_allgather) == pack + ncclAllGather, on 2
    ranks (skipped on a single-GPU box; the driver's 1-GPU test run cannot exercise it)."""
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29631",
                        os.path.join(root, "tools", "gpu", "peer_gather_check.py")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "PEER_GATHER_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
