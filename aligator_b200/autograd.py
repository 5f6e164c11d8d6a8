"""``torch.autograd`` entry point of the batched LQ solve: gradients of the solution with respect to the problem
data, by one adjoint sweep on the device (``ab2_gar_adjoint``, include/aligator_b200/gar.h), and forward-mode
derivatives along a data tangent, by one tangent sweep (``ab2_gar_tangent``).

    xs, us, vs, vsT, lam0, lams = lq_solve(batch, stage, term, G0, g0, mueq)

``batch`` is a plain serial :class:`aligator_b200.gar.CudaRiccatiBatch`; ``stage`` [batch][N][stage_record],
``term`` [batch][term_record], ``G0`` [batch][nc0*nx] and ``g0`` [batch][nc0] are contiguous float64 CUDA tensors
in the layouts of gar.h.  :func:`stage_records` and :func:`term_records` build them differentiably from blocks.

Q and R are symmetric, and their gradient is the one with respect to a symmetric argument (Q_ij and Q_ji perturbed
together).  That is the right chain rule when Q and R are built symmetric, e.g. as ``(P + P^T) / 2`` or ``L L^T``.
Forward mode (``torch.func.jvp``, ``torch.autograd.forward_ad``) is its exact transpose: the tangent of Q and R enters
through ``sym(Qdot) = (Qdot + Qdot^T) / 2``, so an asymmetric tangent acts as its symmetric part.  ``jacfwd`` and
``vmap`` are not supported: the function has no vmap rule.  The penalty ``mueq`` (a number or a [batch] tensor) is not
differentiated.
"""
from __future__ import annotations

import torch
from torch._C import _functorch

from . import gar as _gar

_OUTS = (_gar.OUT_XS, _gar.OUT_US, _gar.OUT_VS, _gar.OUT_VST, _gar.OUT_LBD0, _gar.OUT_LBDAS)
_KEYS = ("xs", "us", "vs", "vsT", "lam0", "lams")
_INPUTS = ("stage", "term", "G0", "g0")


def _input_shapes(batch):
    d = batch.dims
    return dict(stage=(d.batch, d.horizon, batch.srec), term=(d.batch, batch.trec), G0=(d.batch, d.nc0 * d.nx),
                g0=(d.batch, d.nc0))


def _check_inputs(batch, arrays):
    if not isinstance(batch, _gar.CudaRiccatiBatch):
        raise ValueError("lq_solve: `batch` must be a CudaRiccatiBatch")
    for name, shape in _input_shapes(batch).items():
        t = arrays[name]
        if not isinstance(t, torch.Tensor):
            raise ValueError("lq_solve: %s must be a torch tensor" % name)
        if t.dtype != torch.float64 or not t.is_cuda or not t.is_contiguous() or tuple(t.shape) != shape:
            raise ValueError("lq_solve: %s must be a contiguous float64 CUDA tensor of shape %s (got %s %s %s%s)"
                             % (name, shape, t.dtype, t.device, tuple(t.shape),
                                "" if t.is_contiguous() else ", non-contiguous"))


def _outputs(batch, device, stream):
    """The handle's trajectory outputs copied into new tensors."""
    outs = []
    for w in _OUTS:
        t = torch.empty(batch.out_shape(w), dtype=torch.float64, device=device)
        if t.numel():
            batch.get_into(w, _plain(t), _gar.AB2_DEVICE, stream=stream)
        outs.append(t)
    return tuple(outs)


def _plain(t):
    """The tensor beneath torch.func's transform wrappers (itself when it is not wrapped)."""
    while _functorch.is_functorch_wrapped_tensor(t):
        t = _functorch.get_unwrapped(t)
    return t


class _LqSolve(torch.autograd.Function):
    @staticmethod
    def forward(batch, stage, term, G0, g0, mueq):
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        batch.sweep(mueq, stream=stream)
        return _outputs(batch, stage.device, stream)

    @staticmethod
    def setup_context(ctx, inputs, output):
        batch, stage, term, G0, g0, mueq = inputs
        ctx.batch, ctx.mueq = batch, mueq
        ctx.save_for_backward(stage, term, G0, g0, *output)
        ctx.save_for_forward(stage, term, G0, g0, *output)
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *gouts):
        stage, term, G0, g0, *outs = ctx.saved_tensors
        inputs = dict(zip(_INPUTS, (stage, term, G0, g0)))
        grads = {k: torch.empty_like(t) for i, (k, t) in enumerate(inputs.items()) if ctx.needs_input_grad[1 + i]}
        if grads and any(g is not None for g in gouts):
            batch = ctx.batch
            stream = torch.cuda.current_stream(stage.device).cuda_stream
            batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
            cot = {k: None if g is None else g.to(torch.float64).contiguous() for k, g in zip(_KEYS, gouts)}
            batch.adjoint(dict(zip(_KEYS, outs)), cot, grads, ctx.mueq, stream=stream)
        else:
            grads = {}
        return (None,) + tuple(grads.get(k) for k in _INPUTS) + (None,)

    @staticmethod
    def jvp(ctx, _batch_t, *tangents):
        # under torch.func.jvp the saved tensors and tangents arrive wrapped; the library needs the storage beneath
        stage, term, G0, g0, *outs = [_plain(t) for t in ctx.saved_tensors]
        batch = ctx.batch
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        dot = {k: None if t is None else _plain(t.to(torch.float64).contiguous())
               for k, t in zip(_INPUTS, tangents[:4])}
        if all(t is None for t in dot.values()):
            return tuple(torch.zeros_like(o) for o in outs)
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        batch.tangent(dict(zip(_KEYS, outs)), dot, ctx.mueq, stream=stream)
        return _outputs(batch, stage.device, stream)


def lq_solve(batch, stage, term, G0, g0, mueq):
    """Solve the batch's LQ problems on ``torch.cuda.current_stream()``; returns ``(xs, us, vs, vsT, lam0, lams)``
    in the solver's output layouts, differentiable with respect to ``stage``, ``term``, ``G0`` and ``g0``.
    Raises ``ValueError`` before any library call on a tensor that is not a contiguous float64 CUDA tensor of the
    handle's shape."""
    _check_inputs(batch, dict(stage=stage, term=term, G0=G0, g0=g0))
    return _LqSolve.apply(batch, stage, term, G0, g0, mueq)


def _colmajor(M):
    """[..., m, n] blocks -> [..., m*n] in column-major order (the records' storage order)."""
    return M.transpose(-1, -2).reshape(*M.shape[:-2], M.shape[-2] * M.shape[-1])


def stage_records(A, B, f, Q, S, R, q, r, C, D, d):
    """Stage records [..., stage_record] = [A | B | f | Q | S | R | q | r | C | D | d | pad to even] from blocks with
    any leading dimensions (typically [batch, N]): A [..., nx, nx], B [..., nx, nu], f [..., nx], Q [..., nx, nx],
    S [..., nx, nu], R [..., nu, nu], q [..., nx], r [..., nu], C [..., nc, nx], D [..., nc, nu], d [..., nc].
    Differentiable; the pad entry is a constant zero."""
    parts = [_colmajor(A), _colmajor(B), f, _colmajor(Q), _colmajor(S), _colmajor(R), q, r, _colmajor(C),
             _colmajor(D), d]
    rec = torch.cat(parts, dim=-1)
    if rec.shape[-1] % 2:
        rec = torch.cat([rec, rec.new_zeros(*rec.shape[:-1], 1)], dim=-1)
    return rec


def term_records(Q, q, C, d):
    """Terminal records [..., term_record] = [Q | q | C | d] from Q [..., nx, nx], q [..., nx], C [..., nct, nx],
    d [..., nct].  Differentiable."""
    return torch.cat([_colmajor(Q), q, _colmajor(C), d], dim=-1)
