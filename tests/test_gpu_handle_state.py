"""What the solver handle holds after each call (DESIGN §1, "Handle state"): after every state-changing call, which
gated calls refuse with AB2_ERR_STATE, and how factor_epoch and the factor ring head move."""
import ctypes as C

import numpy as np
import pytest

import gen
from inner_cases import random_fddp

pytestmark = pytest.mark.gpu

FIELDS = ("problem", "current", "backward", "primal_factor", "forward", "primal")
# call -> (fields it sets; "primal": None = the value of primal_factor, epoch delta); DESIGN §1's table
TABLE = {
    "set_problem": (dict(problem=True, current=False), 1),
    "assemble": (dict(problem=True, current=False), 1),
    "backward": (dict(current=True, backward=True, primal_factor=True, forward=False, primal=False), 1),
    "sweep": (dict(current=True, backward=True, primal_factor=True, forward=True, primal=True), 1),
    "forward": (dict(forward=True, primal=None), 0),
    "sweep_host": (dict(problem=True, current=True, backward=True, primal_factor=True, forward=True, primal=True), 1),
    "adjoint": (dict(current=True, backward=True, primal_factor=False, forward=True, primal=False), 1),
    "tangent": (dict(current=True, backward=True, primal_factor=False, forward=True, primal=False), 1),
    "cycle_append": (dict(current=False, backward=False, forward=False, primal=False), 1),
    "fddp_backward_pass": (dict(problem=True, current=True, backward=True, primal_factor=True, forward=False,
                                primal=False), 2),
}
# gated call -> what it needs
GATES = {
    "resolve": lambda f: f["problem"] and f["current"],
    "factor_adjoint": lambda f: f["problem"] and f["current"] and f["primal_factor"],
    "refine": lambda f: f["problem"] and f["current"] and f["primal"],
    "kkt_error": lambda f: f["problem"] and f["backward"] and f["forward"],
    "get_gains": lambda f: f["backward"],
    "first_step_policy": lambda f: f["backward"],
    "directional_derivative": lambda f: f["forward"],
}
SCRIPT = ["set_problem", "backward", "forward", "adjoint", "forward", "tangent", "sweep", "cycle_append",
          "cycle_append", "sweep_host", "cycle_append", "assemble", "sweep", "fddp_backward_pass",
          "set_problem"]


@pytest.mark.parametrize("kind", [dict(), dict(variant=9)], ids=["warp", "cta"])
def test_transition_table(kind):
    import torch
    import aligator_b200.gar as gar
    nx, nu, N, B = 12, 6, 5, 4
    L = gar.lib()
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B, **kind)
    stage, term, G0, g0 = gar.pack_problems(gen.generate_batch(5, B, N, nx, nu))
    dev = lambda a: torch.tensor(np.ascontiguousarray(a), device="cuda")
    zeros = lambda *shape: torch.zeros(shape, dtype=torch.float64, device="cuda")
    sol = dict(xs=(B, N + 1, nx), us=(B, N, nu), vs=(B, N, 0), vsT=(B, 0), lam0=(B, nx), lams=(B, N, nx))
    cm = lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2))
    fd = random_fddp(np.random.default_rng(2), B, N, nx, nu)
    fddp = {k: dev(cm(v) if v.ndim >= 3 and k not in ("fs", "Lx", "Lu", "Lx_N") else v) for k, v in fd.items()}
    lq = {k: fddp[k] for k in ("Jx", "Ju", "Lxx", "Lxu", "Luu", "Lx", "Lu", "Lxx_N", "Lx_N")}
    lq.update(slack=fddp["fs"][:, 1:].contiguous(), G0=dev(np.tile(-np.eye(nx).ravel(), (B, 1))),
              g0=fddp["fs"][:, 0].contiguous())
    primal = {k: zeros(*v) for k, v in sol.items()}
    mu = 1e-3
    calls = {
        "set_problem": lambda: s.set_problem(stage, term, G0, g0),
        "assemble": lambda: s.assemble(lq, 1e-4, 1.0),
        "backward": lambda: s.backward(mu),
        "sweep": lambda: s.sweep(mu),
        "forward": lambda: s.forward(),
        "sweep_host": lambda: (s.sweep_host(stage, term, G0, g0, mu, {}), s.synchronize()),
        "adjoint": lambda: s.adjoint(primal, {}, {}, mu),
        "tangent": lambda: s.tangent(primal, {}, mu),
        "cycle_append": lambda: s.cycle_append(stage[:, 0]),
        "fddp_backward_pass": lambda: s.fddp_backward_pass(fddp, 1e-4),
    }
    out1, out2, out3 = np.empty((B, 3)), np.empty(B * N * (nx + nu) * (nx + 1)), np.empty(B)
    pol, Lxs, Lus = zeros(B, nu, nx + 1), zeros(B, N + 1, nx), zeros(B, N, nu)
    null_rhs, null_sol = gar.LqRhs(), gar._fill(gar.LsIterate(), gar._LS_KEYS, primal)
    null_cot, null_grad = gar.FactorCotangent(), gar.LqGrad()
    probes = {  # each call's return code; none of them changes what the handle holds
        "resolve": lambda: L.ab2_gar_resolve(s.h, mu, 0, C.byref(null_rhs), C.byref(null_sol), None),
        "factor_adjoint": lambda: L.ab2_gar_factor_adjoint(s.h, mu, C.byref(null_cot), C.byref(null_grad), None),
        "refine": lambda: L.ab2_gar_refine(s.h, mu, 0, None, None),
        "kkt_error": lambda: L.ab2_gar_kkt_error(s.h, mu, gar._ptr(out1), gar.AB2_HOST, None),
        "get_gains": lambda: L.ab2_gar_get_gains(s.h, gar._ptr(out2), gar.AB2_HOST, None),
        "first_step_policy": lambda: L.ab2_gar_first_step_policy(s.h, gar._ptr(pol), None),
        "directional_derivative": lambda: L.ab2_gar_directional_derivative(s.h, gar._ptr(Lxs), gar._ptr(Lus),
                                                                           gar._ptr(out3), gar.AB2_HOST, None),
    }

    def heads():
        fh, sh = C.c_int(), C.c_int()
        assert L.ab2_gar_ring_heads(s.h, C.byref(fh), C.byref(sh)) == 0
        return fh.value, sh.value

    flags = dict.fromkeys(FIELDS, False)
    for name, probe in probes.items():  # a new handle holds nothing
        assert probe() == 4, name
    for step, call in enumerate(SCRIPT):
        e0, (f0, s0) = s.factor_epoch(), heads()
        calls[call]()
        sets, de = TABLE[call]
        for k, v in sets.items():
            flags[k] = flags["primal_factor"] if v is None else v
        assert s.factor_epoch() == e0 + de, (step, call)
        fh, sh = heads()
        if call == "cycle_append":  # both rings advance (the records are the handle's own copy here)
            assert (fh, sh) == ((f0 + 1) % N, (s0 + 1) % N), (step, call)
        else:  # a backward rewrites every factor slot in knot order; new records are in knot order
            new_records = call in ("set_problem", "assemble", "sweep_host", "fddp_backward_pass")
            assert (fh, sh) == (0 if sets.get("backward") else f0, 0 if new_records else s0), (step, call)
        for name, probe in probes.items():
            want = 0 if GATES[name](flags) else 4
            assert probe() == want, (step, call, name, flags)
        torch.cuda.synchronize()
    s.close()
