"""CPU execution of the CUDA group program (riccati_group.cuh) through the host
emulation (tests/emu_harness.py: G threads + a barrier per group), compared
with the oracle.  This validates the kernel's arithmetic and indexing without a
GPU; the TMA/mbarrier plumbing is the only part it cannot see."""
import numpy as np
import pytest

import gen
from emu_harness import check_against_oracle, emulate
from oracle import gar_oracle as orc


@pytest.mark.parametrize("db", [0, 1])
@pytest.mark.parametrize("shape", [
    (2, 2, 0, 0, 8), (6, 3, 0, 0, 20), (12, 6, 0, 0, 12), (14, 7, 0, 0, 6), (10, 4, 0, 0, 10),
    (3, 2, 0, 0, 9), (8, 3, 0, 0, 7)])
def test_emulated_kernel_unconstrained(shape, db):
    nx, nu, nc, nct, N = shape
    check_against_oracle(nx, nu, nc, nct, N, B=3, mueq=1e-8, seed=sum(shape), db=db)


@pytest.mark.parametrize("shape,mueq", [
    ((4, 2, 2, 0, 25), 1e-3), ((4, 2, 2, 0, 25), 1e-6), ((2, 2, 2, 0, 8), 1e-4),
    ((5, 2, 2, 0, 10), 1e-3), ((12, 6, 6, 0, 8), 1e-3)])
@pytest.mark.parametrize("db", [0, 1])
def test_emulated_kernel_constrained(shape, mueq, db):
    """Constrained knots: D = I rows with a random half inactive (2x2 pivots and
    interchanges occur); gated at the mueq values of SURVEY §8(d)."""
    nx, nu, nc, nct, N = shape
    check_against_oracle(nx, nu, nc, nct, N, B=4, mueq=mueq, seed=7 + sum(shape), db=db)


def test_emulated_kernel_terminal_constraints():
    """Terminal knot with nct > 0 (Z = C/mu branch, riccati-kernel.hxx:146-149)."""
    check_against_oracle(4, 2, 2, 3, 12, B=2, mueq=1e-3, seed=5, tol=1e-9)
    check_against_oracle(6, 3, 0, 2, 10, B=2, mueq=1e-2, seed=6, tol=1e-9)


def test_emulated_kernel_horizon_zero_and_one():
    check_against_oracle(4, 2, 0, 0, 0, B=2, mueq=1e-8, seed=1)
    check_against_oracle(4, 2, 0, 0, 1, B=2, mueq=1e-8, seed=2)


def test_emulated_kernel_reference_style_unstable_A():
    """A ~ U[-1,1] (reference generator style): still within 1e-10 for nc = 0."""
    check_against_oracle(6, 3, 0, 0, 40, B=2, mueq=1e-8, seed=3, style="reference")


@pytest.mark.parametrize("db", [0, 1])
@pytest.mark.parametrize("shape", [(6, 3, 0, 0, 12), (12, 6, 0, 0, 8), (2, 2, 0, 0, 6)])
def test_emulated_kernel_unconstrained_with_interchanges(shape, db):
    """Rhat needs pivoting although nc = 0: the branch-free fast path must detect it and
    fall back to the general Bunch-Kaufman (same results as the oracle)."""
    nx, nu, nc, nct, N = shape
    probs = gen.make_pivoting(gen.generate_batch(31, 2, N, nx, nu, nc, nct))
    # the oracle really does pivot on these problems
    op = orc.OracleProblem(probs[0])
    ref = orc.ProximalRiccatiSolver(op)
    ref.backward(1e-8)
    piv = np.concatenate([ref.factor(t)["bk_piv"] for t in range(N)])
    ident = np.concatenate([np.arange(nu) for _ in range(N)])
    assert np.any(piv != ident)
    check_against_oracle(nx, nu, nc, nct, N, B=2, mueq=1e-8, seed=31, db=db, pivoting=True, tol=1e-9)


@pytest.mark.parametrize("db", [2, 3])
@pytest.mark.parametrize("shape", [(12, 6, 0, 0, 10), (14, 7, 0, 0, 5), (10, 4, 0, 0, 6)])
def test_emulated_tensor_core_step(shape, db):
    """db=2: the DMMA (mma.sync m8n8k4 f64) formulation of the stage step, with the mma
    emulated by a fragment exchange between the 32 lane-threads; db=3: the same with a
    single record buffer refilled in two parts."""
    nx, nu, nc, nct, N = shape
    check_against_oracle(nx, nu, nc, nct, N, B=2, mueq=1e-8, seed=17 + nx, db=db)


def test_emulated_tensor_core_step_with_interchanges():
    check_against_oracle(12, 6, 0, 0, 8, B=2, mueq=1e-8, seed=31, db=2, pivoting=True, tol=1e-9)


@pytest.mark.parametrize("db", [2, 3])
def test_emulated_tensor_core_step_edge_horizons(db):
    check_against_oracle(12, 6, 0, 0, 0, B=1, mueq=1e-8, seed=3, db=db)
    check_against_oracle(12, 6, 0, 0, 1, B=1, mueq=1e-8, seed=4, db=db)
    check_against_oracle(12, 6, 0, 2, 4, B=1, mueq=1e-2, seed=5, db=db, tol=1e-9)


def test_pivot_statistics_and_initial_fast_path():
    """ab2_gar_pivot_stats semantics in the emulation: well-posed problems take the register fast path
    of the initial saddle system and no 2x2 pivot; make_2x2_pivots() problems take min(nu,nc) 2x2
    pivots per knot; make_pivoting() problems take one interchange per knot."""
    nx, nu, N, B = 12, 6, 6, 3
    pivots_2x2 = lambda o: o["pivstat"] & 0x7fff
    interchanges = lambda o: (o["pivstat"] >> 16) & 0xffff
    got = emulate("group", gen.generate_batch(3, B, N, nx, nu, 0, 0), (nx, nu, 0, 0, N), 1e-8, 2)
    kkt0_fast = ((got["pivstat"] >> 15) & 1).astype(bool)
    assert np.all(kkt0_fast) and np.all(pivots_2x2(got) == 0) and np.all(interchanges(got) == 0)
    got = emulate("group", gen.make_pivoting(gen.generate_batch(3, B, N, nx, nu, 0, 0)), (nx, nu, 0, 0, N), 1e-8, 2)
    assert np.all(interchanges(got) >= N)
    nx, nu, nc = 4, 2, 2
    probs = gen.make_2x2_pivots(gen.generate_batch(4, B, N, nx, nu, nc, 0))
    got = emulate("group", probs, (nx, nu, nc, 0, N), 1e-3, 1)
    assert np.all(pivots_2x2(got) >= N * min(nu, nc))
    got["Vxx"] = got["Vxx"].reshape(B, N + 1, nx, nx).transpose(0, 1, 3, 2)
    stage, term, G0, g0 = gen.pack_problems(probs)
    bo = orc.BatchedOracle(nx, nu, nc, 0, nx, N, B, stage, term, G0, g0)
    bo.sweep(1e-3)
    ref = bo.get()
    for k in ("fb", "ff", "Vxx", "xs", "us", "vs", "lbdas"):
        assert gen.rel_fro(got[k], ref[k]) <= 1e-10, k


@pytest.mark.parametrize("shape,db", [((12, 6, 0, 0, 6), 2), ((6, 3, 0, 0, 5), 0), ((4, 2, 2, 0, 4), 1)])
def test_in_sweep_exchange_of_the_first_step_policy(shape, db):
    """Sharded batch (SURVEY 8e): with SweepParams::peer_* set, the sweep itself stores every instance's
    [K_0 | k_0] (nu x (nx+1), row-major) into slot [rank] of EVERY rank's receive buffer at peer_off --
    here three host buffers stand in for the peer-mapped ones.  Everything else in the buffers stays
    untouched, and the sweep's own outputs are unchanged."""
    nx, nu, nc, nct, N = shape
    B, world, rank, slot = 3, 3, 1, 2
    probs = gen.generate_batch(5, B, N, nx, nu, nc, nct)
    per = nu * (nx + 1)
    total = B * per
    bufs = [np.full(3 * world * total, -7.0) for _ in range(world)]
    off = slot * world * total + rank * total
    out = emulate("group", probs, shape, 1e-6, db, peers=(bufs, off))
    ref = emulate("group", probs, shape, 1e-6, db)
    assert np.array_equal(out["fb"], ref["fb"]) and np.array_equal(out["xs"], ref["xs"])
    want = np.concatenate([out["fb"][:, 0, :nu, :], out["ff"][:, 0, :nu, None]], axis=2).ravel()
    for b in bufs:
        assert np.array_equal(b[off:off + total], want)
        assert np.all(b[:off] == -7.0) and np.all(b[off + total:] == -7.0)
