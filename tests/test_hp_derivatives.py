"""The derivatives of the LQ solve against extended-precision references (tests/hp_reference.py), on the CPU.

The references: the forward mode of every output of the sweep by central differences of the 100-digit recursion
(`hp.tangent_problem`), and the reverse modes of the solution and of the factorisation by the closed forms of
tests/lq_adjoint_ref.py and tests/lq_factor_adjoint_ref.py evaluated on object arrays.  Here:
- the closed forms are pinned to the central differences entry by entry on a tiny problem, and by duality
  <g, pdot> = <cbar, ydot(pdot)> on every case, to 1e-25;
- the fp64 restatements, fed with the oracle's factorisation and solution, are measured against the references: their
  error e_ref is the bar of every implementation, and it is set beside the error of the fp64 torch derivation of the
  factorisation's derivatives (test_factor_adjoint_oracle.torch_factor);
- the device programs compiled for the host (factor_adjoint_emu, factor_tangent_emu; resolve_emu followed by the
  restatements' streaming step, the CPU stand-in for adjoint_many / tangent_many) meet the bar of DESIGN §5:
  e_kernel <= max(16 e_ref, 64 u) family by family, each family's error the worst per-(instance, knot) relative error;
- the bar rejects a 1e-12 relative error in one entry of one knot that the 1e-10 batch-Frobenius comparisons accept."""
import functools

import numpy as np
import pytest

import gen
import hp_reference as hp
import lq_adjoint_ref as aref
import lq_factor_adjoint_ref as fadj
import lq_factor_tangent_ref as ftan
import lq_tangent_ref as tref
import test_factor_adjoint_oracle as tfa
import test_factor_tangent_oracle as tft
import test_resolve_oracle as tro
from oracle import gar_oracle as orc
from test_jacobian_oracle import _cot_rhs, grad_many

PIN = 1e-25  # the closed forms against the central differences

# name: ((nx, nu, nc, nct, nc0, N), batch, mu, transform)
CASES = {
    "c3_mu1e-3": ((4, 2, 2, 2, 4, 8), 2, 1e-3, None),
    "c3_mu1e-8": ((4, 2, 2, 2, 4, 8), 2, 1e-8, None),
    "c3_mu1e-11": ((4, 2, 2, 0, 4, 10), 2, 1e-11, None),
    "c2_nct3_mu1e-8": ((12, 6, 0, 3, 12, 4), 2, 1e-8, None),
    "c1": ((6, 3, 0, 2, 3, 5), 2, 1e-3, None),
    "pad_nc0_1": ((4, 2, 1, 1, 1, 5), 2, 1e-3, None),
    "pivots_2x2": ((4, 2, 2, 2, 4, 6), 2, 1e-3, gen.make_2x2_pivots),
    "interchanges": ((6, 3, 0, 0, 6, 6), 2, 1e-3, gen.make_pivoting),
    "nc0_0": ((4, 2, 2, 2, 0, 5), 2, 1e-3, None),
    "N0": ((4, 2, 2, 2, 4, 0), 2, 1e-3, None),
    "N1": ((6, 3, 0, 2, 3, 1), 2, 1e-3, None),
}


def make_problems(name, seed=4000):
    (nx, nu, nc, nct, nc0, N), B, mu, transform = CASES[name]
    probs = gen.generate_batch(seed + sum(map(ord, name)), B, N, nx, nu, nc, nct)
    gen.general_initial_condition(probs, nc0, 7)
    if transform is not None:
        transform(probs)
    return probs


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
        test_factor_adjoint_oracle.torch_factor)."""
        st, tt = self.recs[0], self.recs[1]
        B = tt.shape[0]
        mus = np.broadcast_to(np.asarray(self.mu, dtype=np.float64), (B,))
        one = lambda d, b: {k: v[b:b + 1] for k, v in d.items()}
        per = [(tfa._autograd(st[b:b + 1], tt[b:b + 1], self.d6, mus[b], one(self.fcot, b))[1],
                tft._jvp(st[b:b + 1], tt[b:b + 1], self.d6, mus[b],
                         dict(stage=self.dot["stage"][b:b + 1], term=self.dot["term"][b:b + 1]))[1]) for b in range(B)]
        ga, jv = ({k: np.concatenate([p[i][k] for p in per]) for k in per[0][i]} for i in (0, 1))
        ga.update(G0=np.zeros((B, self.d6[4] * self.d6[0])), g0=np.zeros((B, self.d6[4])))
        return dict(factor_adjoint=self.e_factor_adjoint(ga), factor_tangent=self.e_factor_tangent(jv))


@functools.lru_cache(maxsize=None)
def case(name):
    return Case(make_problems(name), CASES[name][2])


def check_bar(e_kernel, e_ref, title, e_torch=None):
    """e_kernel <= max(16 e_ref, 64 u) family by family; the table of the case on failure."""
    bad = hp.violations(e_kernel, e_ref)
    assert not bad, hp.table(title, e_ref, e_kernel, e_torch)


# ---------------------------------------------------------------------------------------------------------------------
# The closed forms, pinned
# ---------------------------------------------------------------------------------------------------------------------
def _unit_direction(key, shape, idx, d6):
    """The data direction of one record entry; a Q or R entry (i, j) moves along (E_ij + E_ji) / 2, the symmetric
    argument's convention of the gradient records."""
    nx, nu, nc, nct, nc0, N = d6
    d = np.zeros(shape)
    d[idx] = 1.0
    offs = {"stage": (aref.stage_offsets(nx, nu, nc)[0], (("Q", nx), ("R", nu))),
            "term": (aref.term_offsets(nx, nct)[0], (("Q", nx),))}
    if key in offs:
        off, blocks = offs[key]
        for blk, m in blocks:
            a, b = off[blk]
            if a <= idx[-1] < b:
                i, j = (idx[-1] - a) % m, (idx[-1] - a) // m
                if i != j:
                    d[idx] = 0.5
                    d[idx[:-1] + (a + j + i * m,)] = 0.5
    return d


def _pairing(y, c, keys):
    return hp.MP.fsum(hp.MP.fsum(np.ravel(y[k] * c[k])) for k in keys if np.size(c[k]))


def test_closed_forms_match_central_differences_entry_by_entry():
    """Every entry of the extended-precision adjoint and factor-adjoint records is the central difference of the
    100-digit recursion along that entry, to 1e-25 (the fp64 anchors of the formulas stop at 1e-6); the pad double and
    the factor adjoint's G0 and g0 are exactly zero."""
    d6 = (4, 2, 2, 2, 4, 2)
    nx, nu, nc, nct, nc0, N = d6
    probs = gen.general_initial_condition(gen.generate_batch(4100, 1, N, nx, nu, nc, nct), nc0, 5)
    mu = 1e-3
    rng = np.random.default_rng(2)
    cot = {k: rng.standard_normal(s) for k, s in aref._shapes(d6, 1).items()}
    fcot = fadj.random_cot(rng, d6, 1)
    _, hps = hp.solve(probs, mu)
    g = hp.grad_solution(probs, mu, cot, hps)
    gf = hp.grad_factor(probs, mu, fcot, hps)
    assert not gf["G0"].any() and not gf["g0"].any()
    so, srec = aref.stage_offsets(nx, nu, nc)
    assert np.all(g["stage"][..., so["d"][1]:] == 0) and np.all(gf["stage"][..., so["d"][1]:] == 0)
    worst = {"adjoint": 0.0, "factor_adjoint": 0.0}
    for key, arr in zip(("stage", "term", "G0", "g0"), hp.records(probs)):
        for idx in np.ndindex(*arr.shape):
            if key == "stage" and idx[-1] >= so["d"][1]:
                continue  # the pad double is no datum
            td = hp.tangent_problem(probs[0], mu, {key: _unit_direction(key, arr.shape, idx, d6)[0]})
            sol = {k: v[None] for k, v in hp.solution_of(td).items()}
            fac = {k: v[None] for k, v in hp.factor_of(td).items()}
            for what, want, an in (("adjoint", _pairing(sol, cot, aref.KEYS), g[key][idx]),
                                   ("factor_adjoint", _pairing(fac, fcot, fadj.COT), gf[key][idx])):
                worst[what] = max(worst[what], float(abs(want - an) / max(abs(an), 1)))
    assert max(worst.values()) <= PIN, worst


@pytest.mark.parametrize("name", list(CASES))
def test_closed_forms_satisfy_duality_with_the_central_differences(name):
    """<g_hp, pdot> = <cbar, ydot_hp(pdot)> to 1e-25 for three random directions, for the solution's and the
    factorisation's gradients."""
    c = case(name)
    probs, mu, d6 = c.probs, c.mu, c.d6
    g = hp.grad_solution(probs, mu, c.cot, c.hps)
    gf = hp.grad_factor(probs, mu, c.fcot, c.hps)
    rng = np.random.default_rng(3)
    for _ in range(3):
        dot = symmetric_dot(rng, d6, len(probs))
        _, td = hp.tangents(probs, mu, dot)
        zd = hp.solution_dict(td)
        fd = {k: np.stack([hp.factor_of(t)[k] for t in td]) for k in fadj.COT}
        for lhs, rhs in ((_pairing(zd, c.cot, aref.KEYS), _pairing(g, dot, g)),
                         (_pairing(fd, c.fcot, fadj.COT), _pairing(gf, dot, gf))):
            scale = max(abs(lhs), abs(rhs), 1)
            assert abs(lhs - rhs) <= PIN * scale, (name, float(lhs), float(rhs))


# ---------------------------------------------------------------------------------------------------------------------
# The fp64 restatements against the references: e_ref
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_restatements_against_extended_precision(name):
    """The restatements fed by the oracle (the bar every implementation is held to) are finite everywhere and never
    more than 16 times worse than the fp64 torch derivation of the factorisation's derivatives.  (Measured: 1e-15 to
    9e-12 per (instance, knot) at mu = 1e-3, 1e-11 at mu = 1e-8 times the problems' 1 / mu; DESIGN §5.)"""
    c = case(name)
    e_ref, e_torch = c.e_refs(), c.e_torch()
    for call, e in e_ref.items():
        print("\n" + hp.table("%s %s (e_ref in the e_kernel column)" % (name, call), {f: hp.FLOOR for f in e}, e,
                              e_torch.get(call)))
        assert all(np.isfinite(v) for v in e.values()), (call, e)
    for call, et in e_torch.items():
        worse = {f: (e_ref[call][f], et[f]) for f in et if e_ref[call][f] > hp.FACTOR * max(et[f], hp.FLOOR)}
        assert not worse, (call, worse)


# ---------------------------------------------------------------------------------------------------------------------
# The device programs, emulated on the host, at the bar
# ---------------------------------------------------------------------------------------------------------------------
# (lanes, packed Vxx, ring head): a warp item with packed Vxx, a 7-lane item with full Vxx, a rotated ring
GEOMETRIES = [(32, True, 0), (7, False, 0), (32, True, 3)]
EMU_CASES = [n for n in CASES if n != "c3_mu1e-11"] + ["c3_mu1e-11"]


@pytest.mark.parametrize("name", EMU_CASES)
def test_emulated_factor_programs_meet_the_bar(name):
    c = case(name)
    e_ref = c.e_refs()
    recs, fac, d6, mu = c.recs, c.fac, c.d6, c.mu
    for lanes, packed, head in GEOMETRIES:
        g = tfa.run_emu(recs, fac, c.fcot, d6, mu, lanes, packed, head)
        assert np.isfinite(g["stage"]).all() and not g["G0"].any() and not g["g0"].any()
        geo = (lanes, packed, head)
        check_bar(c.e_factor_adjoint(g), e_ref["factor_adjoint"], "%s factor_adjoint %s" % (name, geo))
        t = tft.run_emu(recs, fac, dict(stage=c.dot["stage"], term=c.dot["term"]), d6, mu, lanes, packed, head)
        check_bar(c.e_factor_tangent(t), e_ref["factor_tangent"], "%s factor_tangent %s" % (name, geo))


def test_emulated_factor_programs_per_instance_mu():
    """Per-instance mu spanning 1e-8 .. 1e-1 through the programs' mu array."""
    probs = make_problems("c3_mu1e-3", 4200)[:2] + make_problems("c3_mu1e-3", 4300)[:2]
    mus = np.array([1e-8, 1e-5, 1e-3, 1e-1])
    c = Case(probs, mus)
    e_ref = c.e_refs()
    for lanes, packed, head in GEOMETRIES[:2]:
        g = tfa.run_emu(c.recs, c.fac, c.fcot, c.d6, mus, lanes, packed, head)
        check_bar(c.e_factor_adjoint(g), e_ref["factor_adjoint"], "factor_adjoint per-instance mu")
        t = tft.run_emu(c.recs, c.fac, dict(stage=c.dot["stage"], term=c.dot["term"]), c.d6, mus, lanes, packed, head)
        check_bar(c.e_factor_tangent(t), e_ref["factor_tangent"], "factor_tangent per-instance mu")


@pytest.mark.parametrize("name", ["c3_mu1e-3", "c3_mu1e-8", "c2_nct3_mu1e-8", "pad_nc0_1", "pivots_2x2", "N0", "N1"])
def test_emulated_many_rhs_meets_the_bar(name):
    """adjoint_many and tangent_many on the host: resolve_emu on the oracle's factorisation for the cotangent (resp.
    rho = Kdot z + hdot), then the streaming kernels' formulas (test_jacobian_oracle.grad_many)."""
    c = case(name)
    e_ref = c.e_refs()
    B = len(c.probs)
    rho = tref.rho(c.dot, c.z, c.d6)
    for lanes, chunk, packed, head in ((32, 2, True, 0), (5, 1, False, 1)):
        y = tro._run_emu(c.recs, c.out, {k: v[None] for k, v in _cot_rhs(c.cot).items()}, c.d6, 1, c.mu, lanes, chunk,
                         packed, head)
        g = grad_many(c.z, {k: v[0] for k, v in y.items()}, c.d6)
        g["G0"], g["g0"] = g["G0"].reshape(B, -1), g["g0"].reshape(B, -1)
        check_bar(c.e_adjoint(g), e_ref["adjoint"], "%s adjoint_many (host) %s" % (name, (lanes, chunk)))
        zd = tro._run_emu(c.recs, c.out, {k: v[None] for k, v in _cot_rhs(rho).items()}, c.d6, 1, c.mu, lanes, chunk,
                          packed, head)
        check_bar(c.e_tangent({k: v[0] for k, v in zd.items()}), e_ref["tangent"],
                  "%s tangent_many (host) %s" % (name, (lanes, chunk)))


# ---------------------------------------------------------------------------------------------------------------------
# Sharpness
# ---------------------------------------------------------------------------------------------------------------------
def _bump(arr, sl):
    """A copy of arr with the largest entry of arr[sl] off by a relative 1e-12."""
    out = np.array(arr, copy=True)
    blk = out[sl]
    i = np.unravel_index(np.argmax(np.abs(blk)), blk.shape)
    blk[i] *= 1 + 1e-12
    assert not np.array_equal(out, arr)
    return out


@pytest.mark.parametrize("name", ["pivots_2x2", "interchanges"])
def test_bar_rejects_a_1e12_error_that_1e10_accepts(name):
    """One entry of one knot's block of a gradient record (the factor adjoint's A, then its Q) and of a factor tangent
    (K), off by a relative 1e-12 in the emulated programs' otherwise correct outputs: the bar rejects it, the 1e-10
    batch-Frobenius comparisons of the GPU tests accept it.  (On cases whose restatements are within ~1e-14.)"""
    c = case(name)
    e_ref = c.e_refs()
    nx, nu, nc, nct, nc0, N = c.d6
    so, _ = aref.stage_offsets(nx, nu, nc)
    t = N // 2
    g = tfa.run_emu(c.recs, c.fac, c.fcot, c.d6, c.mu, 32)
    assert not hp.violations(c.e_factor_adjoint(g), e_ref["factor_adjoint"])
    for fam in ("A", "Q"):
        bad = dict(g, stage=_bump(g["stage"], np.s_[0, t, so[fam][0]:so[fam][1]]))
        assert max(tfa.block_errors(bad, c.gf_ref, c.d6).values()) <= 1e-10
        assert fam in hp.violations(c.e_factor_adjoint(bad), e_ref["factor_adjoint"]), fam
    ft = tft.run_emu(c.recs, c.fac, dict(stage=c.dot["stage"], term=c.dot["term"]), c.d6, c.mu, 32)
    assert not hp.violations(c.e_factor_tangent(ft), e_ref["factor_tangent"])
    bad = dict(ft, fb=_bump(ft["fb"], np.s_[0, t, :nu]))
    assert max(tft.family_errors(bad, c.fd_ref).values()) <= 1e-10
    assert "K" in hp.violations(c.e_factor_tangent(bad), e_ref["factor_tangent"])
