"""CPU execution of the CTA-per-instance sweep for run-time dimensions
(riccati_block.cuh) through tests/emu/block_emu.cpp, compared with the oracle."""
import pytest

from emu_harness import check_against_oracle


@pytest.mark.parametrize("shape,nw", [
    ((7, 3, 0, 0, 6), 1), ((9, 5, 0, 0, 5), 2), ((13, 4, 0, 0, 4), 3), ((20, 9, 0, 0, 3), 2),
    ((1, 1, 0, 0, 4), 1), ((8, 8, 0, 0, 4), 2)])
def test_block_unconstrained_shapes_not_instantiated(shape, nw):
    nx, nu, nc, nct, N = shape
    check_against_oracle(nx, nu, nc, nct, N, B=2, mueq=1e-8, seed=3 + sum(shape), block=nw)


@pytest.mark.parametrize("shape,mueq,nw", [
    ((7, 3, 3, 0, 6), 1e-3, 2), ((9, 4, 4, 0, 5), 1e-4, 2), ((6, 6, 6, 2, 4), 1e-3, 1),
    ((5, 2, 1, 0, 5), 1e-6, 1)])
def test_block_constrained(shape, mueq, nw):
    nx, nu, nc, nct, N = shape
    check_against_oracle(nx, nu, nc, nct, N, B=2, mueq=mueq, seed=11 + sum(shape), block=nw, tol=1e-9)


def test_block_interchanges_and_edge_horizons():
    check_against_oracle(9, 5, 0, 0, 5, B=2, mueq=1e-8, seed=31, block=2, pivoting=True, tol=1e-9)
    check_against_oracle(7, 3, 0, 0, 0, B=1, mueq=1e-8, seed=1, block=1)
    check_against_oracle(7, 3, 0, 0, 1, B=1, mueq=1e-8, seed=2, block=1)
    check_against_oracle(7, 3, 0, 3, 2, B=1, mueq=1e-2, seed=2, block=1, tol=1e-9)


def test_block_wide_kkt_more_than_one_warp_of_rows():
    """nu + nc = 40 > 32 rows in the reduced KKT matrix, nx + nc0 = 48 rows in the
    initial-stage system: one THREAD per row over two warps."""
    check_against_oracle(24, 20, 20, 0, 2, B=1, mueq=1e-3, seed=5, block=2, tol=1e-9)


def test_block_compile_time_specialisation():
    """The same block program instantiated with compile-time dimensions (what BASELINE config 5
    runs on the GPU): block < 0 selects it."""
    check_against_oracle(7, 3, 0, 0, 6, B=2, mueq=1e-8, seed=40, block=-2)
    check_against_oracle(9, 5, 3, 0, 5, B=2, mueq=1e-3, seed=41, block=-2, tol=1e-9)
    check_against_oracle(7, 3, 0, 0, 5, B=1, mueq=1e-8, seed=31, block=-1, pivoting=True, tol=1e-9)


def test_block_random_shapes():
    """Seeded random sweep over run-time shapes (odd sizes, constrained and not, terminal constraints,
    every warp count that fits): catches index arithmetic that only breaks off the beaten path."""
    import numpy as np
    rng = np.random.default_rng(2024)
    done = 0
    while done < 16:
        nx, nu = int(rng.integers(1, 15)), int(rng.integers(1, 9))
        nc = int(rng.integers(0, 4)) if rng.random() < 0.5 else 0
        nct = int(rng.integers(0, 3)) if rng.random() < 0.3 else 0
        N = int(rng.integers(0, 6))
        need = max(nx + 1, nu + nc, 2 * nx, nu + nc + nx)
        nw = int(rng.integers((need + 31) // 32, 4))
        if 32 * nw < need:
            continue
        mueq = 1e-3 if (nc or nct) else 1e-8
        check_against_oracle(nx, nu, nc, nct, N, B=1, mueq=mueq, seed=300 + done, block=nw,
                             tol=1e-9 if (nc or nct) else 1e-10)
        done += 1
