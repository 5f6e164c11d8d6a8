"""Iterative refinement of the LQ solve on the CPU (ab2_gar_refine, gar.h): the numpy restatement of the residual
(lq_refine_ref.py) against K z + h of the dense KKT system, and refinement on the oracle's factorisation with
lq_resolve_ref.resolve as the correction solver against the extended-precision solve (DESIGN §5)."""
import numpy as np
import pytest

import gen
import hp_reference as hp
import lq_refine_ref as fref
import lq_resolve_ref as rref
from lq_cases import BAR_CASES, batch_records, errors, refine_case, refined_on_oracle, run_oracle

# (nx, nu, nc, nct, nc0, N): C1, C2 and C3 dims, nct in {0, 2}, nc0 in {0, 1, nx/2, nx}, N in {0, 1, 5, 100}
CASES = [(6, 3, 0, 0, 6, 5), (6, 3, 0, 2, 1, 1), (12, 6, 0, 0, 12, 1), (12, 6, 0, 2, 6, 0), (12, 6, 0, 0, 0, 5),
         (4, 2, 2, 2, 4, 100), (4, 2, 2, 0, 2, 5), (4, 2, 2, 2, 0, 0), (4, 2, 2, 0, 1, 100), (4, 2, 2, 2, 2, 1)]
IDS = ["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d" % c for c in CASES]
MU = 1e-2


def _probs(case, seed, B=2):
    nx, nu, nc, nct, nc0, N = case
    return gen.general_initial_condition(gen.generate_batch(seed, B, N, nx, nu, nc, nct), nc0, seed)


def _dense_order(p, z, b, j, N):
    """Solution dict entry (rhs j, instance b) -> the unknown vector of gen.lqr_dense_kkt."""
    parts = [z["lam0"][j, b]]
    for t in range(N):
        parts += [z["xs"][j, b, t], z["us"][j, b, t], z["vs"][j, b, t], z["lams"][j, b, t]]
    parts += [z["xs"][j, b, N], z["vsT"][j, b]]
    return np.concatenate(parts)


def _rows_dense_order(r, b, j, N):
    """Residual dict (resolve's rhs layouts) -> the row order of gen.lqr_dense_kkt."""
    parts = [r["g0"][j, b]]
    for t in range(N):
        parts += [r["q"][j, b, t], r["r"][j, b, t], r["d"][j, b, t], r["f"][j, b, t]]
    parts += [r["q"][j, b, N], r["dN"][j, b]]
    return np.concatenate(parts)


@pytest.mark.parametrize("own", [True, False], ids=["own_vectors", "rhs"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_residual_matches_dense_kkt(case, own):
    nx, nu, nc, nct, nc0, N = case
    probs = _probs(case, 21)
    B, nrhs = len(probs), (1 if own else 2)
    stage, term, G0, g0 = batch_records(probs, case)
    rng = np.random.default_rng(22)
    z = {k: rng.standard_normal((nrhs,) + s) for k, s in zip(rref.SOL, rref.rhs_shapes(case, B).values())}
    h = None if own else rref.random_rhs(rng, case, B, nrhs)
    mu = np.array([MU, 3 * MU])
    r = fref.residual(stage, term, G0, g0, z, h, case, mu)
    for b in range(B):
        for j in range(nrhs):
            p = probs[b] if own else rref.replaced_problems([probs[b]], {k: v[j][b:b + 1] for k, v in h.items()})[0]
            K, rhs, _ = gen.lqr_dense_kkt(p, mu[b])
            zv = _dense_order(p, z, b, j, N)
            want = K @ zv + rhs
            got = _rows_dense_order(r, b, j, N)
            scale = np.abs(K).sum(axis=1).max() * np.abs(zv).max() + np.abs(rhs).max()
            assert np.abs(got - want).max() <= 1e-14 * scale, (b, j, np.abs(got - want).max() / scale)
    norms = fref.inf_norms(r)
    assert norms.shape == (nrhs, B) and np.all(norms > 0)


REFINE_CASES = list(BAR_CASES) + ["general_G0"]


@pytest.mark.parametrize("name", REFINE_CASES)
def test_two_steps_reach_the_fp64_floor(name):
    """After two refinement steps on the oracle's factorisation every trajectory family is within max(16 floor, 64 u)
    of the extended-precision solve, and the residual norm has not grown.  The floor is what an fp64 residual allows
    on this factorisation; the cases below show where it is 64 u."""
    probs, recs, case, mu = refine_case(name)
    z, z0, norms, want, floor = refined_on_oracle(probs, recs, case, mu)
    e = errors(z, want, case)
    bad = {f: (e[f], floor[f]) for f in e if not e[f] <= max(16 * floor[f], hp.FLOOR)}
    assert not bad, (name, bad, errors(z0, want, case))
    assert np.all(norms[..., -1] <= norms[..., 0]), norms


@pytest.mark.parametrize("name", ["c3_mu1e-11", "c3_nct_mu1e-8"])
def test_refinement_recovers_lost_digits(name):
    """Where the unrefined trajectory misses 64 u (mu = 1e-11; terminal constraints at mu = 1e-8, where it is good to
    8 digits only), two steps bring every family within 64 u: the test above discriminates."""
    probs, recs, case, mu = refine_case(name)
    z, z0, _, want, _ = refined_on_oracle(probs, recs, case, mu)
    assert max(errors(z0, want, case).values()) > hp.FLOOR
    assert max(errors(z, want, case).values()) <= hp.FLOOR


def test_zero_steps_and_resolve_outputs():
    """refine(0) leaves z alone; refining a resolve output with its own right-hand side changes it by at most a few
    ulps of the solution (resolve is already accurate at mu = 1e-2)."""
    case = (4, 2, 2, 2, 4, 5)
    probs = _probs(case, 23)
    recs = batch_records(probs, case)
    o = run_oracle(recs, case, MU)
    h = rref.random_rhs(np.random.default_rng(24), case, 2, 3)
    z0 = rref.resolve(recs[0], recs[1], recs[2], o["fb"], o["fbT"], o["Vxx"], h, case, MU, 3)
    z, norms = fref.refine(*recs, o["fb"], o["fbT"], o["Vxx"], z0, h, case, MU, 0)
    assert norms.shape == (3, 2, 1)
    for k in z:
        assert np.array_equal(z[k], z0[k])
    z, norms = fref.refine(*recs, o["fb"], o["fbT"], o["Vxx"], z0, h, case, MU, 2)
    for k in z:
        assert gen.rel_fro(z[k], z0[k]) <= 1e-12, k
