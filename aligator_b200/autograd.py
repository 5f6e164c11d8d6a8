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
through ``sym(Qdot) = (Qdot + Qdot^T) / 2``, so an asymmetric tangent acts as its symmetric part.  The penalty
``mueq`` (a number or a [batch] tensor) is not differentiated, and the gradients and jvps are not differentiable again.

Jacobians: under ``torch.func.jacrev``, ``jacfwd``, ``vmap`` of a vjp function or ``vmap`` over ``torch.func.jvp``
tangents, the V cotangents or tangents go to the device in one call on one factorisation (``ab2_gar_adjoint_many`` /
``ab2_gar_tangent_many``, through ``ab2_gar_resolve``; one single call per slice on a dense handle).  Outside vmap the
gradients and jvps are those of one ``adjoint`` or ``tangent`` call.  vmap over the problem data itself raises
``NotImplementedError``.

:func:`lq_factor` returns the factorisation of the backward pass -- gains ``ff``, ``fb`` and cost-to-go ``vxx``, ``vx``,
``fft``, ``fbt`` -- differentiable with respect to ``stage`` and ``term`` by one reverse pass of the matrix recursion
on the device (``ab2_gar_factor_adjoint``).  Reverse mode only (``jacrev`` works, one device call per cotangent);
G0 and g0 do not enter the factorisation.  :func:`lq_factor_fwd` returns the same outputs, bit for bit,
differentiable in forward mode instead (``torch.func.jvp``, ``forward_ad``, ``jacfwd``) by one tangent pass of the
matrix recursion on the device (``ab2_gar_factor_tangent``) per tangent: the cheap direction for the whole gain
schedule's sensitivity to a few parameters.

:func:`lq_resolve` re-solves the matrices of the handle's last backward for new vectors (``ab2_gar_resolve``), many
right-hand sides in one call.  It is linear in the vectors and its own transpose, so its ``backward`` and ``jvp`` are
``lq_resolve`` calls again, and it has a vmap rule: ``torch.func.vmap``, ``jacrev``, ``jacfwd`` and higher orders work
with respect to the vectors.

:func:`lq_solve_higher` returns ``lq_solve``'s outputs, bit for bit, differentiable to any order (gradient penalties,
Hessian-vector products, ``torch.func.hessian``): every derivative is resolve plus the two stateless streaming maps
``ab2_gar_rho_many`` and ``ab2_gar_grad_many`` (DESIGN section 2p), through four Functions whose backward, jvp and vmap
rules call each other.  ``lq_solve`` itself stays differentiable once.

:func:`lq_solve_theta` solves a parametric problem (nth > 0) at ``theta`` and is differentiable with respect to theta,
in both modes and to any order: the solution is affine in theta, and its Jacobian J is applied from the stored factors
by ``ab2_gar_theta_tangent`` (J d) and ``ab2_gar_theta_adjoint`` (J^T zbar), one launch per vmap level.
"""
from __future__ import annotations

import torch
from torch._C import _functorch
from torch.autograd.function import once_differentiable

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
        need = tuple(ctx.needs_input_grad[1:5])
        if not any(need) or all(g is None for g in gouts):
            return (None,) * 6
        grads = iter(_LqSolveVjp.apply(ctx.batch, ctx.mueq, need, stage, term, G0, g0, *outs, *gouts))
        return (None,) + tuple(next(grads) if n else None for n in need) + (None,)

    @staticmethod
    def jvp(ctx, _batch_t, *tangents):
        # under torch.func.jvp the saved tensors arrive wrapped; the library needs the storage beneath.  The tangents
        # are passed on as they are: under vmap (jacfwd) they are batched, and _LqSolveJvp's vmap rule takes them.
        stage, term, G0, g0, *outs = [_plain(t) for t in ctx.saved_tensors]
        dot = tangents[:4]
        if all(t is None for t in dot):
            return tuple(torch.zeros_like(o) for o in outs)
        return _LqSolveJvp.apply(ctx.batch, ctx.mueq, stage, term, G0, g0, *outs, *dot)

    @staticmethod
    def vmap(info, in_dims, batch, stage, term, G0, g0, mueq):
        # torch runs the forward unbatched when no input is batched (jacfwd, vmap over cotangents); it needs this rule
        # to exist all the same
        raise NotImplementedError(_NO_DATA_VMAP)


_NO_DATA_VMAP = ("lq_solve: vmap over the problem data (stage, term, G0, g0, mueq) is not supported; vmap over "
                 "cotangents and tangents is (torch.func.jacrev, jacfwd, vmap of a vjp or jvp function)")
_NOT_TWICE = "lq_solve is differentiable once: its gradients and jvps have no derivatives"


def _stacked(t, bd, V):
    """A vmapped argument as a [V][...] float64 tensor: its batch dimension first, or broadcast when unbatched."""
    if t is None:
        return None
    t = t.movedim(bd, 0) if bd is not None else t.unsqueeze(0).expand(V, *t.shape)
    return t.to(torch.float64).contiguous()


class _LqSolveVjp(torch.autograd.Function):
    """Gradient records of ``lq_solve`` for the cotangents ``gouts`` of its outputs: one ``adjoint`` call, or under vmap
    one ``adjoint_many`` over all the cotangents (one ``adjoint`` per cotangent on a dense handle)."""

    @staticmethod
    def forward(batch, mueq, need, stage, term, G0, g0, *rest):
        # saved tensors of a torch.func.vjp arrive as wrappers of a finished transform; the library needs the storage
        stage, term, G0, g0, *outs = [_plain(t) for t in (stage, term, G0, g0) + rest[:6]]
        gouts = rest[6:]
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        inputs = dict(zip(_INPUTS, (stage, term, G0, g0)))
        grads = {k: torch.empty_like(t) for (k, t), n in zip(inputs.items(), need) if n}
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        cot = {k: None if g is None else g.to(torch.float64).contiguous() for k, g in zip(_KEYS, gouts)}
        batch.adjoint(dict(zip(_KEYS, outs)), cot, grads, mueq, stream=stream)
        return tuple(grads.values())

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    @once_differentiable
    def backward(ctx, *_):
        raise RuntimeError(_NOT_TWICE)

    @staticmethod
    def vmap(info, in_dims, batch, mueq, need, stage, term, G0, g0, *rest):
        if any(d is not None for d in (in_dims[1],) + in_dims[3:13]):  # in_dims[2]: `need`, not a tensor
            raise NotImplementedError(_NO_DATA_VMAP)
        V = info.batch_size
        stage, term, G0, g0, *outs = [_plain(t) for t in (stage, term, G0, g0) + rest[:6]]
        primal = dict(zip(_KEYS, outs))
        cot = {k: _stacked(g, bd, V) for k, g, bd in zip(_KEYS, rest[6:], in_dims[13:])}
        shapes = {k: t.shape for k, t in zip(_INPUTS, (stage, term, G0, g0))}
        grads = {k: torch.empty((V,) + shapes[k], dtype=torch.float64, device=stage.device)
                 for k, n in zip(_INPUTS, need) if n}
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        if batch.dense:  # resolve does not serve dense handles: one adjoint per cotangent
            for j in range(V):
                batch.adjoint(primal, {k: None if c is None else c[j] for k, c in cot.items()},
                              {k: g[j] for k, g in grads.items()}, mueq, stream=stream)
        else:
            batch.backward(mueq, stream=stream)
            work = {k: torch.empty((V,) + o.shape, dtype=torch.float64, device=stage.device) for k, o in primal.items()}
            batch.adjoint_many(primal, cot, work, grads, mueq, stream=stream)
        return tuple(grads.values()), 0


class _LqSolveJvp(torch.autograd.Function):
    """The derivative of ``lq_solve``'s outputs along the data tangents ``dot``: one ``tangent`` call, or under vmap one
    ``tangent_many`` over all the tangents (one ``tangent`` per tangent on a dense handle)."""

    @staticmethod
    def forward(batch, mueq, stage, term, G0, g0, *rest):
        outs, dot = rest[:6], rest[6:]
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        dot = {k: None if t is None else _plain(t.to(torch.float64).contiguous()) for k, t in zip(_INPUTS, dot)}
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        batch.tangent(dict(zip(_KEYS, outs)), dot, mueq, stream=stream)
        return _outputs(batch, stage.device, stream)

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    @once_differentiable
    def backward(ctx, *_):
        raise RuntimeError(_NOT_TWICE)

    @staticmethod
    def vmap(info, in_dims, batch, mueq, stage, term, G0, g0, *rest):
        if any(d is not None for d in in_dims[1:12]):
            raise NotImplementedError(_NO_DATA_VMAP)
        V = info.batch_size
        stage, term, G0, g0, *outs = [_plain(t) for t in (stage, term, G0, g0) + rest[:6]]
        primal = dict(zip(_KEYS, outs))
        dot = {k: _stacked(t, bd, V) for k, t, bd in zip(_INPUTS, rest[6:], in_dims[12:])}
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        if batch.dense:  # resolve does not serve dense handles: one tangent per tangent
            res = []
            for j in range(V):
                batch.tangent(primal, {k: None if t is None else t[j] for k, t in dot.items()}, mueq, stream=stream)
                res.append(_outputs(batch, stage.device, stream))
            return tuple(torch.stack(r) for r in zip(*res)), 0
        batch.backward(mueq, stream=stream)
        work = {k: torch.empty((V,) + o.shape, dtype=torch.float64, device=stage.device) for k, o in primal.items()}
        res = {k: torch.empty((V,) + o.shape, dtype=torch.float64, device=stage.device) for k, o in primal.items()}
        batch.tangent_many(primal, dot, work, res, mueq, stream=stream)
        return tuple(res[k] for k in _KEYS), 0


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


_RHS = ("q", "r", "d", "dN", "g0", "f")


def _rhs_shapes(batch):
    """Per-right-hand-side shape of each vector field, in the layouts of the solution (q like xs, ..., f like lams)."""
    d = batch.dims
    B, N = d.batch, d.horizon
    return dict(q=(B, N + 1, d.nx), r=(B, N, d.nu), d=(B, N, d.nc), dN=(B, d.nct), g0=(B, d.nc0), f=(B, N, d.nx))


class _LqResolve(torch.autograd.Function):
    """z = resolve(h) on [nrhs][batch][...] tensors.  Linear and self-transpose: VJP and JVP are resolve again."""

    @staticmethod
    def forward(batch, mueq, epoch, *h):
        if batch.factor_epoch() != epoch:
            raise RuntimeError("lq_resolve: the handle has been refactored since these derivatives were recorded")
        h = [None if t is None else _plain(t).to(torch.float64).contiguous() for t in h]
        given = [t for t in h if t is not None]
        device = given[0].device if given else torch.device("cuda", batch.dims.device)
        nrhs = given[0].shape[0] if given else 1
        outs = [torch.empty((nrhs,) + s, dtype=torch.float64, device=device) for s in _rhs_shapes(batch).values()]
        if nrhs:
            stream = torch.cuda.current_stream(device).cuda_stream
            batch.resolve(dict(zip(_RHS, h)), dict(zip(_KEYS, outs)), mueq, stream=stream)
        return tuple(outs)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.batch, ctx.mueq, ctx.epoch = inputs[:3]
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *gz):
        if all(g is None for g in gz):
            return (None,) * 9
        gh = _LqResolve.apply(ctx.batch, ctx.mueq, ctx.epoch, *gz)
        return (None, None, None) + tuple(g if need else None for g, need in zip(gh, ctx.needs_input_grad[3:]))

    @staticmethod
    def jvp(ctx, _b, _m, _e, *hdot):
        return _LqResolve.apply(ctx.batch, ctx.mueq, ctx.epoch, *hdot)

    @staticmethod
    def vmap(info, in_dims, batch, mueq, epoch, *h):
        V = info.batch_size
        flat = []
        for t, bd in zip(h, in_dims[3:]):
            if t is not None:
                t = t.movedim(bd, 0) if bd is not None else t.unsqueeze(0).expand(V, *t.shape)
                t = t.reshape(V * t.shape[1], *t.shape[2:])
            flat.append(t)
        outs = _LqResolve.apply(batch, mueq, epoch, *flat)
        return tuple(o.reshape(V, o.shape[0] // V, *o.shape[1:]) for o in outs), (0,) * len(outs)


def lq_resolve(batch, mueq, q=None, r=None, d=None, dN=None, g0=None, f=None):
    """Solve the LQ problem of ``batch``'s last backward with its vectors replaced by (q, r, d, dN, g0, f); returns
    ``(xs, us, vs, vsT, lam0, lams)``.  Each vector has the shape of the solution field it pairs with (q like xs
    [batch][N+1][nx], r like us, d like vs, dN like vsT, g0 like lam0 [batch][nc0], f like lams with f_t in the row of
    lambda_{t+1}) behind any leading dimensions; the leading dimensions are broadcast, flattened into the right-hand
    sides of one device call, and lead every output.  None is zero.  ``mueq`` must be the mu of that backward.
    Differentiable with respect to the vectors in both modes and under ``torch.func`` transforms; calling ``backward``
    or ``jvp`` after the handle has been refactored (``factor_epoch`` changed) raises RuntimeError."""
    if not isinstance(batch, _gar.CudaRiccatiBatch):
        raise ValueError("lq_resolve: `batch` must be a CudaRiccatiBatch")
    shapes = _rhs_shapes(batch)
    h = dict(q=q, r=r, d=d, dN=dN, g0=g0, f=f)
    lead = []
    for k, t in h.items():
        if t is None:
            continue
        s = shapes[k]
        if not isinstance(t, torch.Tensor) or t.dim() < len(s) or tuple(t.shape[t.dim() - len(s):]) != s:
            raise ValueError("lq_resolve: %s must be a tensor of shape [..., %s]" % (k, ", ".join(map(str, s))))
        lead.append(tuple(t.shape[:t.dim() - len(s)]))
    lead = tuple(torch.broadcast_shapes(*lead)) if lead else ()
    nrhs = 1
    for n in lead:
        nrhs *= n
    flat = [None if t is None else t.expand(*lead, *shapes[k]).reshape(nrhs, *shapes[k]) for k, t in h.items()]
    outs = _LqResolve.apply(batch, mueq, batch.factor_epoch(), *flat)
    return tuple(o.reshape(*lead, *o.shape[1:]) for o in outs)


_FOUTS = (_gar.OUT_FF, _gar.OUT_FB, _gar.OUT_VXX, _gar.OUT_VX, _gar.OUT_FFT, _gar.OUT_FBT)
_FKEYS = ("ff", "fb", "vxx", "vx", "fft", "fbt")
_NO_FACTOR_DATA_VMAP = ("lq_factor: vmap over the problem data (stage, term, G0, g0, mueq) is not supported; vmap "
                        "over cotangents is (torch.func.jacrev, vmap of a vjp function)")
_NO_FACTOR_JVP = ("lq_factor: forward mode of the gains is not supported (torch.func.jvp, jacfwd, forward_ad); use "
                  "reverse mode (backward, torch.func.vjp, jacrev), or lq_factor_fwd for forward mode")


def _factor_cotangent(gouts):
    """Cotangents of lq_factor's outputs -> device layouts: vxx back to column-major blocks."""
    cot = {}
    for k, g in zip(_FKEYS, gouts):
        if g is not None:
            g = g.to(torch.float64)
            if k == "vxx":
                g = g.transpose(-1, -2)
            g = g.contiguous()
        cot[k] = g
    return cot


def _factor_outputs(batch, stage, term, G0, g0, mueq):
    """Set the problem, run the backward pass and copy the factorisation out: the outputs of lq_factor and
    lq_factor_fwd."""
    stream = torch.cuda.current_stream(stage.device).cuda_stream
    batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
    batch.backward(mueq, stream=stream)
    outs = []
    for w in _FOUTS:
        t = torch.empty(batch.out_shape(w), dtype=torch.float64, device=stage.device)
        if t.numel():
            batch.get_into(w, t, _gar.AB2_DEVICE, stream=stream)
        outs.append(t.transpose(-1, -2).contiguous() if w == _gar.OUT_VXX else t)  # VXX blocks are column-major
    return tuple(outs)


class _LqFactor(torch.autograd.Function):
    @staticmethod
    def forward(batch, stage, term, G0, g0, mueq):
        return _factor_outputs(batch, stage, term, G0, g0, mueq)

    @staticmethod
    def setup_context(ctx, inputs, output):
        batch, stage, term, G0, g0, mueq = inputs
        ctx.batch, ctx.mueq = batch, mueq
        ctx.save_for_backward(stage, term, G0, g0)
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *gouts):
        stage, term, G0, g0 = ctx.saved_tensors
        need = tuple(ctx.needs_input_grad[1:3])
        if not any(need) or all(g is None for g in gouts):
            return (None,) * 6
        grads = iter(_LqFactorVjp.apply(ctx.batch, ctx.mueq, need, stage, term, G0, g0, *gouts))
        return (None,) + tuple(next(grads) if n else None for n in need) + (None,) * 3

    @staticmethod
    def jvp(ctx, *_):
        raise NotImplementedError(_NO_FACTOR_JVP)

    @staticmethod
    def vmap(info, in_dims, batch, stage, term, G0, g0, mueq):
        raise NotImplementedError(_NO_FACTOR_DATA_VMAP)


class _LqFactorVjp(torch.autograd.Function):
    """Gradient records (stage, term) of ``lq_factor`` for the cotangents ``gouts`` of its outputs: a backward, then one
    ``factor_adjoint`` call, or under vmap one ``factor_adjoint`` call per cotangent on that backward."""

    @staticmethod
    def forward(batch, mueq, need, stage, term, G0, g0, *gouts):
        stage, term, G0, g0 = [_plain(t) for t in (stage, term, G0, g0)]
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        grads = {k: torch.empty_like(t) for (k, t), n in zip((("stage", stage), ("term", term)), need) if n}
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        batch.backward(mueq, stream=stream)
        batch.factor_adjoint(_factor_cotangent(gouts), grads, mueq, stream=stream)
        return tuple(grads.values())

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    @once_differentiable
    def backward(ctx, *_):
        raise RuntimeError("lq_factor is differentiable once: its gradients have no derivatives")

    @staticmethod
    def vmap(info, in_dims, batch, mueq, need, stage, term, G0, g0, *gouts):
        if any(d is not None for d in (in_dims[1],) + in_dims[3:7]):  # in_dims[2]: `need`, not a tensor
            raise NotImplementedError(_NO_FACTOR_DATA_VMAP)
        V = info.batch_size
        stage, term, G0, g0 = [_plain(t) for t in (stage, term, G0, g0)]
        cot = [_stacked(g, bd, V) for g, bd in zip(gouts, in_dims[7:])]
        grads = {k: torch.empty((V,) + t.shape, dtype=torch.float64, device=stage.device)
                 for (k, t), n in zip((("stage", stage), ("term", term)), need) if n}
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        batch.backward(mueq, stream=stream)
        for j in range(V):
            batch.factor_adjoint(_factor_cotangent([None if c is None else c[j] for c in cot]),
                                 {k: g[j] for k, g in grads.items()}, mueq, stream=stream)
        return tuple(grads.values()), 0


def lq_factor(batch, stage, term, G0, g0, mueq):
    """Run the backward pass of the batch's LQ problems on ``torch.cuda.current_stream()``; returns the factorisation
    ``(ff, fb, vxx, vx, fft, fbt)``: ff [batch][N][nu+nc+nx] = [k; z; a], fb [batch][N][nu+nc+nx][nx] = [K; Z; Ahat],
    vxx [batch][N+1][nx][nx] (indexed [b, t, i, j]), vx [batch][N+1][nx], fft [batch][nct] = z_N and fbt
    [batch][nct][nx] = Z_N.  Differentiable in reverse mode with respect to ``stage`` and ``term`` (Q and R as
    symmetric arguments, cotangents of vxx taken through their symmetric part); G0 and g0 do not enter the
    factorisation and get no gradient.  Each backward re-sets the problem and reruns the backward pass, so losses that
    mix ``lq_factor`` and ``lq_solve`` outputs of one handle get the summed gradient in any order.  Forward mode raises
    ``NotImplementedError``.  Raises ``ValueError`` before any library call on a tensor that is not a contiguous float64
    CUDA tensor of the handle's shape."""
    _check_inputs(batch, dict(stage=stage, term=term, G0=G0, g0=g0))
    return _LqFactor.apply(batch, stage, term, G0, g0, mueq)


_NO_FACTOR_FWD_DATA_VMAP = ("lq_factor_fwd: vmap over the problem data (stage, term, G0, g0, mueq) is not supported; "
                            "vmap over tangents is (torch.func.jacfwd, vmap of a jvp function)")
_NO_FACTOR_FWD_BACKWARD = ("lq_factor_fwd is differentiable in forward mode only (torch.func.jvp, jacfwd, forward_ad); "
                           "use lq_factor for reverse mode")


class _LqFactorFwd(torch.autograd.Function):
    @staticmethod
    def forward(batch, stage, term, G0, g0, mueq):
        return _factor_outputs(batch, stage, term, G0, g0, mueq)

    @staticmethod
    def setup_context(ctx, inputs, output):
        batch, stage, term, G0, g0, mueq = inputs
        ctx.batch, ctx.mueq = batch, mueq
        ctx.save_for_forward(stage, term, G0, g0)
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *_):
        raise RuntimeError(_NO_FACTOR_FWD_BACKWARD)

    @staticmethod
    def jvp(ctx, _batch_t, dstage, dterm, _dG0, _dg0, _mueq_t):
        # G0 and g0 do not enter the factorisation.  The tangents are passed on as they are: under vmap (jacfwd) they
        # are batched, and _LqFactorTangent's vmap rule takes them.
        stage, term, G0, g0 = [_plain(t) for t in ctx.saved_tensors]
        return _LqFactorTangent.apply(ctx.batch, ctx.mueq, stage, term, G0, g0, dstage, dterm)

    @staticmethod
    def vmap(info, in_dims, batch, stage, term, G0, g0, mueq):
        # torch runs the forward unbatched when no input is batched (jacfwd); it needs this rule to exist all the same
        raise NotImplementedError(_NO_FACTOR_FWD_DATA_VMAP)


def _factor_tangent_into(batch, mueq, dot, outs, stream):
    """One factor_tangent call: ``outs`` in lq_factor's shapes (vxx [..][i][j]) receive the tangents along ``dot``."""
    dev = dict(zip(_FKEYS, outs))
    vxx = torch.empty_like(dev["vxx"])  # the device writes column-major blocks
    dev["vxx"] = vxx
    batch.factor_tangent(dot, {k: t for k, t in dev.items() if t.numel()}, mueq, stream=stream)
    outs[2].copy_(vxx.transpose(-1, -2))


class _LqFactorTangent(torch.autograd.Function):
    """The derivative of ``lq_factor_fwd``'s outputs along the data tangents ``dstage``, ``dterm``: a backward, then one
    ``factor_tangent`` call, or under vmap one ``factor_tangent`` call per tangent on that backward."""

    @staticmethod
    def forward(batch, mueq, stage, term, G0, g0, dstage, dterm):
        stage, term, G0, g0 = [_plain(t) for t in (stage, term, G0, g0)]
        dot = {k: None if t is None else _plain(t.to(torch.float64).contiguous())
               for k, t in (("stage", dstage), ("term", dterm))}
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        outs = [torch.empty(batch.out_shape(w), dtype=torch.float64, device=stage.device) for w in _FOUTS]
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        batch.backward(mueq, stream=stream)
        _factor_tangent_into(batch, mueq, dot, outs, stream)
        return tuple(outs)

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    @once_differentiable
    def backward(ctx, *_):
        raise RuntimeError("lq_factor_fwd is differentiable once: its jvps have no derivatives")

    @staticmethod
    def vmap(info, in_dims, batch, mueq, stage, term, G0, g0, dstage, dterm):
        if any(d is not None for d in in_dims[2:6]):
            raise NotImplementedError(_NO_FACTOR_FWD_DATA_VMAP)
        V = info.batch_size
        stage, term, G0, g0 = [_plain(t) for t in (stage, term, G0, g0)]
        dot = {k: _stacked(t, bd, V) for k, t, bd in (("stage", dstage, in_dims[6]), ("term", dterm, in_dims[7]))}
        stream = torch.cuda.current_stream(stage.device).cuda_stream
        outs = [torch.empty((V,) + tuple(batch.out_shape(w)), dtype=torch.float64, device=stage.device)
                for w in _FOUTS]
        batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        batch.backward(mueq, stream=stream)
        for j in range(V):
            _factor_tangent_into(batch, mueq, {k: None if t is None else t[j] for k, t in dot.items()},
                                 [o[j] for o in outs], stream)
        return tuple(outs), (0,) * 6


def lq_factor_fwd(batch, stage, term, G0, g0, mueq):
    """:func:`lq_factor`'s outputs, bit for bit, differentiable in FORWARD mode with respect to ``stage`` and ``term``
    (``torch.func.jvp``, ``torch.autograd.forward_ad``, ``jacfwd``): each jvp re-sets the problem, reruns the backward
    pass and makes one ``factor_tangent`` call (under ``jacfwd`` one call per tangent on that backward).  The tangent
    of Q and R enters through its symmetric part; G0 and g0 do not enter the factorisation.  Reverse mode raises
    ``RuntimeError`` (use :func:`lq_factor`), and vmap over the problem data raises ``NotImplementedError``.  Raises
    ``ValueError`` before any library call on a tensor that is not a contiguous float64 CUDA tensor of the handle's
    shape."""
    _check_inputs(batch, dict(stage=stage, term=term, G0=G0, g0=g0))
    return _LqFactorFwd.apply(batch, stage, term, G0, g0, mueq)


# ---- higher derivatives of the solve: lq_solve_higher, from resolve and the two streaming maps (DESIGN section 2p) ----
_NO_HIGHER_HANDLE = ("lq_solve_higher: plain serial handles only (warp and CTA kernels); dense, parametric and parallel "
                     "handles are not served by resolve")


class _Higher:
    """The handle and mu of one lq_solve_higher call, and the factor epoch at which the handle's factorisation is that
    call's data."""

    def __init__(self, batch, mueq):
        self.batch, self.mueq, self.epoch = batch, mueq, None
        self.sol = tuple(tuple(batch.out_shape(w)) for w in _OUTS)
        self.rec = tuple(_input_shapes(batch).values())

    def stream(self, device):
        return torch.cuda.current_stream(device).cuda_stream

    def factor(self, P, stream):
        """Make the handle's factorisation that of the data P = (stage, term, G0, g0), re-running set_problem and
        backward when another call has moved the factor epoch since."""
        if self.batch.factor_epoch() != self.epoch:
            self.batch.set_problem(*P, memspace=_gar.AB2_DEVICE, stream=stream)
            self.batch.backward(self.mueq, stream=stream)
            self.epoch = self.batch.factor_epoch()


def _none(ts):
    return ts is None or all(t is None for t in ts)


def _directions(ts, shapes):
    """The number of directions of the operands ts (base shapes `shapes`): the leading size of those that carry one,
    None when every operand has its base shape."""
    for t, s in zip(ts, shapes):
        if t is not None and t.dim() == len(s) + 1:
            return t.shape[0]
    return None


def _device(h, ts):
    for t in ts:
        if t is not None:
            return t.device
    return torch.device("cuda", h.batch.dims.device)


def _per(t, s, n, device):
    """t as a contiguous float64 [n][...] tensor: broadcast when it has its base shape s, zeros when None."""
    if t is None:
        return torch.zeros((n,) + s, dtype=torch.float64, device=device)
    if t.dim() == len(s):
        t = t.unsqueeze(0).expand(n, *s)
    return t.to(torch.float64).contiguous()


def _vector(ts, shapes, n, device):
    """A vector operand as the library's dict: shared ([batch][...]) when none of its fields carries directions, else
    every field [n][...]; None fields are zeros."""
    if _directions(ts, shapes) is None:
        return {k: (torch.zeros(s, dtype=torch.float64, device=device) if t is None else t.to(torch.float64).contiguous())
                for k, t, s in zip(_KEYS, ts, shapes)}
    return {k: _per(t, s, n, device) for k, t, s in zip(_KEYS, ts, shapes)}


def _records(ts, shapes, n):
    return {k: None if t is None else _per(t, s, n, t.device) for k, t, s in zip(_INPUTS, ts, shapes)}


def _results(outs, n):
    return tuple(o if n else o[0] for o in outs)


def _fold(info, in_dims, args, kinds, refuse):
    """The vmap rule of the higher-order Functions: every vmapped dimension goes into the directions of one call.  An
    operand of kind s (its base shape) that carries the level's dimension and directions of an inner level becomes
    [V * n][...]; one without either is broadcast to them, or stays shared when no operand has inner directions.  Kind
    "P" (the problem data) is refused when vmapped, kind None is passed as it is."""
    V = info.batch_size
    moved = []
    for t, bd, k in zip(args, in_dims, kinds):
        if k == "P" and bd is not None:
            raise NotImplementedError(refuse)
        moved.append(t.movedim(bd, 0) if bd is not None and isinstance(k, tuple) else t)
    n = None
    for t, bd, k in zip(moved, in_dims, kinds):
        if isinstance(k, tuple) and t is not None and t.dim() - (bd is not None) > len(k):
            n = t.shape[1 if bd is not None else 0]
    flat = []
    for t, bd, k in zip(moved, in_dims, kinds):
        if isinstance(k, tuple) and t is not None:
            inner = t.dim() - (bd is not None) > len(k)
            if bd is not None and n is not None:
                t = (t if inner else t.unsqueeze(1).expand(V, n, *k)).reshape(V * n, *k)
            elif bd is None and inner:
                t = t.unsqueeze(0).expand(V, *t.shape).reshape(V * n, *k)
        flat.append(t)
    return flat, n


def _unfold(info, outs, n):
    V = info.batch_size
    return tuple(o.reshape(V, n, *o.shape[1:]) if n else o for o in outs), (0,) * len(outs)


def _rho_sum(h, terms, e):
    """sum of rho^(v)(P; a) over terms (v, P, a) plus e, by _Rho calls of at most two terms each (the term with
    vectors first); terms with a zero P, or a zero a without vectors, are dropped.  None when nothing is left."""
    terms = sorted([t for t in terms if not _none(t[1]) and not (_none(t[2]) and not t[0])], key=lambda t: not t[0])
    none4, none6 = (None,) * 4, (None,) * 6
    while terms:
        first = terms.pop(0)
        second = terms.pop(0) if terms else None
        e = _Rho.apply(h, first[0], *first[1], *(first[2] or none6), *(second[1] if second else none4),
                       *((second[2] or none6) if second else none6), *(e or none6))
    return e


def _grad_sum(h, pairs):
    """sum of Gr^(v)(y; z) over pairs (v, y, z), by _Grad calls of at most two pairs each (the pair with vectors
    first); pairs with a zero y, or a zero z without vectors, are dropped.  None when nothing is left."""
    pairs = sorted([p for p in pairs if not _none(p[1]) and not (_none(p[2]) and not p[0])], key=lambda p: not p[0])
    none6, total = (None,) * 6, None
    while pairs:
        first = pairs.pop(0)
        second = pairs.pop(0) if pairs else None
        g = _Grad.apply(h, first[0], *first[1], *(first[2] or none6), *(second[1] if second else none6),
                        *((second[2] or none6) if second else none6))
        total = g if total is None else tuple(a + b for a, b in zip(total, g))
    return total


def _pick(values, need):
    return tuple(v if n else None for v, n in zip(values, need)) if values is not None else (None,) * len(need)


class _Solve(torch.autograd.Function):
    """z = solve(P): set_problem and sweep.  jvp: resolve(rho(Pdot; z)); vjp: Gr(resolve(c); z)."""

    @staticmethod
    def forward(h, stage, term, G0, g0):
        stream = h.stream(stage.device)
        h.batch.set_problem(stage, term, G0, g0, memspace=_gar.AB2_DEVICE, stream=stream)
        h.batch.sweep(h.mueq, stream=stream)
        h.epoch = h.batch.factor_epoch()
        return _outputs(h.batch, stage.device, stream)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.h = inputs[0]
        ctx.save_for_backward(*inputs[1:], *output)
        ctx.save_for_forward(*inputs[1:], *output)
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *c):
        if _none(c):
            return (None,) * 5
        saved = ctx.saved_tensors
        P, z = saved[:4], saved[4:]
        m = _Resolve.apply(ctx.h, *P, *c)
        return (None,) + _pick(_grad_sum(ctx.h, [(True, m, z)]), ctx.needs_input_grad[1:5])

    @staticmethod
    def jvp(ctx, _h, *Pdot):
        saved = ctx.saved_tensors
        P, z = saved[:4], saved[4:]
        if _none(Pdot):
            return tuple(torch.zeros_like(t) for t in z)
        return _Resolve.apply(ctx.h, *P, *_rho_sum(ctx.h, [(True, Pdot, z)], None))

    @staticmethod
    def vmap(info, in_dims, h, stage, term, G0, g0):
        raise NotImplementedError(_NO_DATA_VMAP)


class _Resolve(torch.autograd.Function):
    """z = resolve_P(h) = -K(P)^-1 h, h in the solution's layouts.  jvp: resolve(hdot + rho_K(Pdot; z)); vjp: hbar =
    m = resolve(c), Pbar = Gr_K(m; z)."""

    @staticmethod
    def forward(h, stage, term, G0, g0, *hv):
        n = _directions(hv, h.sol)
        device = stage.device
        outs = [torch.empty((n or 1,) + s, dtype=torch.float64, device=device) for s in h.sol]
        stream = h.stream(device)
        if _none(hv):
            return _results([o.zero_() for o in outs], n)
        h.factor((stage, term, G0, g0), stream)
        rhs = {k: None if t is None else _per(t, s, n or 1, device) for k, t, s in zip(_RHS, hv, h.sol)}
        h.batch.resolve(rhs, dict(zip(_KEYS, outs)), h.mueq, stream=stream)
        return _results(outs, n)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.h = inputs[0]
        ctx.save_for_backward(*inputs[1:5], *output)
        ctx.save_for_forward(*inputs[1:5], *output)
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *c):
        if _none(c):
            return (None,) * 11
        saved = ctx.saved_tensors
        P, z = saved[:4], saved[4:]
        need = ctx.needs_input_grad
        m = _Resolve.apply(ctx.h, *P, *c)
        Pbar = _grad_sum(ctx.h, [(False, m, z)]) if any(need[1:5]) else None
        return (None,) + _pick(Pbar, need[1:5]) + _pick(m, need[5:])

    @staticmethod
    def jvp(ctx, _h, *dots):
        saved = ctx.saved_tensors
        P, z = saved[:4], saved[4:]
        r = _rho_sum(ctx.h, [(False, dots[:4], z)], None if _none(dots[4:]) else dots[4:])
        if r is None:
            return tuple(torch.zeros_like(t) for t in z)
        return _Resolve.apply(ctx.h, *P, *r)

    @staticmethod
    def vmap(info, in_dims, h, *args):
        flat, n = _fold(info, in_dims[1:], args, ("P",) * 4 + h.sol, _NO_DATA_VMAP)
        return _unfold(info, _Resolve.apply(h, *flat), n)


class _Rho(torch.autograd.Function):
    """r = rho^(vec)(P1; a1) + rho_K(P2; a2) + e (ab2_gar_rho_many), in the solution's layouts.  jvp:
    rho^(vec)(P1'; a1) + rho_K(P1; a1') + rho_K(P2'; a2) + rho_K(P2; a2') + e'; vjp: P1bar = Gr^(vec)(c; a1),
    a1bar = rho_K(P1; c), P2bar = Gr_K(c; a2), a2bar = rho_K(P2; c), ebar = c."""

    @staticmethod
    def forward(h, vec, *args):
        P1, a1, P2, a2, e = args[:4], args[4:10], args[10:14], args[14:20], args[20:26]
        n = _directions(args, h.rec + h.sol + h.rec + h.sol + h.sol)
        device = _device(h, args)
        N = n or 1
        out = {k: torch.empty((N,) + s, dtype=torch.float64, device=device) for k, s in zip(_KEYS, h.sol)}
        two = not _none(P2)
        h.batch.rho_many(_records(P1, h.rec, N), _vector(a1, h.sol, N, device), out, vectors=vec,
                         dot2=_records(P2, h.rec, N) if two else None,
                         a2=_vector(a2, h.sol, N, device) if two else None,
                         e=None if _none(e) else {k: _per(t, s, N, device) for k, t, s in zip(_KEYS, e, h.sol)},
                         stream=h.stream(device))
        return _results(out.values(), n)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.h, ctx.vec = inputs[:2]
        ctx.outs = [(o.shape, o.device) for o in output]
        ctx.save_for_backward(*inputs[2:22])
        ctx.save_for_forward(*inputs[2:22])
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *c):
        if _none(c):
            return (None,) * 28
        saved = ctx.saved_tensors
        P1, a1, P2, a2 = saved[:4], saved[4:10], saved[10:14], saved[14:20]
        need, h = ctx.needs_input_grad[2:], ctx.h
        P1bar = _grad_sum(h, [(ctx.vec, c, a1)]) if any(need[:4]) else None
        a1bar = _rho_sum(h, [(False, P1, c)], None) if any(need[4:10]) else None
        P2bar = _grad_sum(h, [(False, c, a2)]) if any(need[10:14]) else None
        a2bar = _rho_sum(h, [(False, P2, c)], None) if any(need[14:20]) else None
        return ((None, None) + _pick(P1bar, need[:4]) + _pick(a1bar, need[4:10]) + _pick(P2bar, need[10:14])
                + _pick(a2bar, need[14:20]) + _pick(c, need[20:26]))

    @staticmethod
    def jvp(ctx, _h, _vec, *t):
        saved = ctx.saved_tensors
        P1, a1, P2, a2 = saved[:4], saved[4:10], saved[10:14], saved[14:20]
        r = _rho_sum(ctx.h, [(ctx.vec, t[:4], a1), (False, P1, t[4:10]), (False, t[10:14], a2), (False, P2, t[14:20])],
                     None if _none(t[20:26]) else t[20:26])
        return r if r is not None else tuple(torch.zeros(sh, dtype=torch.float64, device=dv) for sh, dv in ctx.outs)

    @staticmethod
    def vmap(info, in_dims, h, vec, *args):
        flat, n = _fold(info, in_dims[2:], args, h.rec + h.sol + h.rec + h.sol + h.sol, _NO_DATA_VMAP)
        return _unfold(info, _Rho.apply(h, vec, *flat), n)


class _Grad(torch.autograd.Function):
    """g = Gr^(vec)(y1; z1) + Gr_K(y2; z2) (ab2_gar_grad_many), in the problem's record layouts.  jvp:
    Gr^(vec)(y1'; z1) + Gr_K(y1; z1') + Gr_K(y2'; z2) + Gr_K(y2; z2'); vjp: y1bar = rho^(vec)(C; z1),
    z1bar = rho_K(C; y1), y2bar = rho_K(C; z2), z2bar = rho_K(C; y2)."""

    @staticmethod
    def forward(h, vec, *args):
        y1, z1, y2, z2 = args[:6], args[6:12], args[12:18], args[18:24]
        n = _directions(args, h.sol * 4)
        device = _device(h, args)
        N = n or 1
        grad = {k: torch.empty((N,) + s, dtype=torch.float64, device=device) for k, s in zip(_INPUTS, h.rec)}
        two = not _none(y2)
        h.batch.grad_many({k: _per(t, s, N, device) for k, t, s in zip(_KEYS, y1, h.sol)},
                          _vector(z1, h.sol, N, device), grad, vectors=vec,
                          y2={k: _per(t, s, N, device) for k, t, s in zip(_KEYS, y2, h.sol)} if two else None,
                          z2=_vector(z2, h.sol, N, device) if two else None, stream=h.stream(device))
        return _results(grad.values(), n)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.h, ctx.vec = inputs[:2]
        ctx.outs = [(o.shape, o.device) for o in output]
        ctx.save_for_backward(*inputs[2:])
        ctx.save_for_forward(*inputs[2:])
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *C):
        if _none(C):
            return (None,) * 26
        saved = ctx.saved_tensors
        y1, z1, y2, z2 = saved[:6], saved[6:12], saved[12:18], saved[18:24]
        need, h = ctx.needs_input_grad[2:], ctx.h
        y1bar = _rho_sum(h, [(ctx.vec, C, z1)], None) if any(need[:6]) else None
        z1bar = _rho_sum(h, [(False, C, y1)], None) if any(need[6:12]) else None
        y2bar = _rho_sum(h, [(False, C, z2)], None) if any(need[12:18]) else None
        z2bar = _rho_sum(h, [(False, C, y2)], None) if any(need[18:24]) else None
        return ((None, None) + _pick(y1bar, need[:6]) + _pick(z1bar, need[6:12]) + _pick(y2bar, need[12:18])
                + _pick(z2bar, need[18:24]))

    @staticmethod
    def jvp(ctx, _h, _vec, *t):
        saved = ctx.saved_tensors
        y1, z1, y2, z2 = saved[:6], saved[6:12], saved[12:18], saved[18:24]
        g = _grad_sum(ctx.h, [(ctx.vec, t[:6], z1), (False, y1, t[6:12]), (False, t[12:18], z2), (False, y2, t[18:24])])
        return g if g is not None else tuple(torch.zeros(sh, dtype=torch.float64, device=dv) for sh, dv in ctx.outs)

    @staticmethod
    def vmap(info, in_dims, h, vec, *args):
        flat, n = _fold(info, in_dims[2:], args, h.sol * 4, _NO_DATA_VMAP)
        return _unfold(info, _Grad.apply(h, vec, *flat), n)


def lq_solve_higher(batch, stage, term, G0, g0, mueq):
    """:func:`lq_solve`'s outputs ``(xs, us, vs, vsT, lam0, lams)``, bit for bit (the same set_problem and sweep),
    differentiable to ANY order with respect to ``stage``, ``term``, ``G0`` and ``g0``: gradient penalties
    (``create_graph=True``), Hessian-vector products (``torch.func.jvp`` of ``torch.func.grad``), ``torch.func.hessian``.
    Every derivative is a composition of resolve (``ab2_gar_resolve``) and the two streaming maps rho and Gr
    (``ab2_gar_rho_many``, ``ab2_gar_grad_many``); under vmap (``jacrev``, ``jacfwd``, ``hessian``) each op makes one
    device call per vmap level, whatever the number of directions.  Its first derivatives equal lq_solve's vmapped ones
    (``jacrev``, ``jacfwd``), and a single vjp or jvp equals ``adjoint_many`` / ``tangent_many`` at nrhs = 1.  A resolve
    runs on the handle's factorisation of this call's data: when another call has refactored the handle since (its
    ``factor_epoch`` moved), set_problem and backward are run again first.  ``mueq`` (a number or a [batch] tensor) is
    not differentiated.  Plain serial handles only: dense, parametric and parallel handles raise ``ValueError`` before
    any library call, as does a tensor that is not a contiguous float64 CUDA tensor of the handle's shape; vmap over the
    problem data raises ``NotImplementedError``."""
    if not isinstance(batch, _gar.CudaRiccatiBatch):
        raise ValueError("lq_solve_higher: `batch` must be a CudaRiccatiBatch")
    if batch.dense or batch.nth > 0 or batch.legs:
        raise ValueError(_NO_HIGHER_HANDLE)
    _check_inputs(batch, dict(stage=stage, term=term, G0=G0, g0=g0))
    return _Solve.apply(_Higher(batch, mueq), stage, term, G0, g0)


# ---------------------------------------------------------------------------------------------------------------------
# Derivatives of a parametric solution with respect to theta
# ---------------------------------------------------------------------------------------------------------------------
_NO_THETA_HANDLE = ("lq_solve_theta: parametric handles only (nth > 0); plain, dense and parallel handles have no theta "
                    "to differentiate")
_NO_THETA_VMAP = ("lq_solve_theta: vmap over theta or the problem data is not supported; vmap over cotangents and "
                  "tangents is (torch.func.jacrev, jacfwd, hessian, vmap of a vjp or jvp function)")


class _Theta(_Higher):
    """The handle, mu and data of one lq_solve_theta call: its factorisation is re-made from the data P when another
    call has moved the factor epoch (_Higher.factor)."""

    def __init__(self, batch, mueq):
        super().__init__(batch, mueq)
        self.P = None
        self.th = (batch.dims.batch, batch.nth)


def _lead(ts, shapes):
    """The broadcast leading dimensions of the operands ts over their base shapes (None operands left out)."""
    leads = [tuple(t.shape[:t.dim() - len(s)]) for t, s in zip(ts, shapes) if t is not None]
    return tuple(torch.broadcast_shapes(*leads)) if leads else ()


def _count(lead):
    n = 1
    for m in lead:
        n *= m
    return n


def _moved(info, t, bd):
    """A vmapped operand with the level's dimension first (broadcast to it when unbatched)."""
    if t is None:
        return None
    return t.movedim(bd, 0) if bd is not None else t.unsqueeze(0).expand(info.batch_size, *t.shape)


class _LqSolveTheta(torch.autograd.Function):
    """z = solve(P, theta): set_problem, backward, forward_theta.  jvp: J thetadot; vjp: J^T zbar."""

    @staticmethod
    def forward(h, stage, term, G0, g0, theta):
        theta = _plain(theta)
        stream = h.stream(theta.device)
        h.P = tuple(_plain(t) for t in (stage, term, G0, g0))
        h.batch.set_problem(*h.P, memspace=_gar.AB2_DEVICE, stream=stream)
        h.batch.backward(h.mueq, stream=stream)
        h.epoch = h.batch.factor_epoch()
        h.batch.forward(stream=stream, theta=theta)
        return _outputs(h.batch, theta.device, stream)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.h = inputs[0]
        ctx.outs = [(o.shape, o.device) for o in output]
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *zbar):
        if _none(zbar):
            return (None,) * 6
        return (None,) * 5 + (_ThetaAdjoint.apply(ctx.h, *zbar),)

    @staticmethod
    def jvp(ctx, _h, _stage, _term, _G0, _g0, dtheta):
        if dtheta is None:
            return tuple(torch.zeros(s, dtype=torch.float64, device=d) for s, d in ctx.outs)
        return _ThetaTangent.apply(ctx.h, dtheta)

    @staticmethod
    def vmap(info, in_dims, h, stage, term, G0, g0, theta):
        # torch runs the forward unbatched when no input is batched (jacfwd, vmap over cotangents); it needs this rule
        # to exist all the same
        raise NotImplementedError(_NO_THETA_VMAP)


class _ThetaTangent(torch.autograd.Function):
    """J d for directions d [..., batch, nth] (ab2_gar_theta_tangent, every leading index one direction).  Linear:
    jvp J ddot, vjp J^T zbar."""

    @staticmethod
    def forward(h, d):
        d = _plain(d)
        lead = tuple(d.shape[:-2])
        n = _count(lead)
        outs = [torch.empty((n,) + s, dtype=torch.float64, device=d.device) for s in h.sol]
        if n:
            stream = h.stream(d.device)
            h.factor(h.P, stream)
            h.batch.theta_tangent(d.reshape(n, *h.th).to(torch.float64).contiguous(), dict(zip(_KEYS, outs)),
                                  stream=stream)
        return tuple(o.reshape(*lead, *o.shape[1:]) for o in outs)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.h = inputs[0]
        ctx.outs = [(o.shape, o.device) for o in output]
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, *zbar):
        if _none(zbar):
            return None, None
        return None, _ThetaAdjoint.apply(ctx.h, *zbar)

    @staticmethod
    def jvp(ctx, _h, ddot):
        if ddot is None:
            return tuple(torch.zeros(s, dtype=torch.float64, device=dv) for s, dv in ctx.outs)
        return _ThetaTangent.apply(ctx.h, ddot)

    @staticmethod
    def vmap(info, in_dims, h, d):
        return _ThetaTangent.apply(h, _moved(info, d, in_dims[1])), (0,) * 6


class _ThetaAdjoint(torch.autograd.Function):
    """J^T zbar for cotangents zbar in the solution's layouts behind any leading dimensions (ab2_gar_theta_adjoint;
    None is zero).  Linear: jvp J^T zdot, vjp J thbar."""

    @staticmethod
    def forward(h, *zbar):
        zbar = [None if t is None else _plain(t) for t in zbar]
        lead = _lead(zbar, h.sol)
        n = _count(lead)
        device = _device(h, zbar)
        tb = torch.empty((n,) + h.th, dtype=torch.float64, device=device)
        if n:
            stream = h.stream(device)
            h.factor(h.P, stream)
            cot = {k: None if t is None else t.expand(*lead, *s).reshape(n, *s).to(torch.float64).contiguous()
                   for k, t, s in zip(_KEYS, zbar, h.sol)}
            h.batch.theta_adjoint(cot, tb, stream=stream)
        return tb.reshape(*lead, *h.th)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.h = inputs[0]
        ctx.out = (output.shape, output.device)
        ctx.set_materialize_grads(False)

    @staticmethod
    def backward(ctx, thbar):
        if thbar is None:
            return (None,) * 7
        return (None,) + _pick(_ThetaTangent.apply(ctx.h, thbar), ctx.needs_input_grad[1:])

    @staticmethod
    def jvp(ctx, _h, *zdot):
        if _none(zdot):
            return torch.zeros(ctx.out[0], dtype=torch.float64, device=ctx.out[1])
        return _ThetaAdjoint.apply(ctx.h, *zdot)

    @staticmethod
    def vmap(info, in_dims, h, *zbar):
        return _ThetaAdjoint.apply(h, *[_moved(info, t, bd) for t, bd in zip(zbar, in_dims[1:])]), 0


def lq_solve_theta(batch, stage, term, G0, g0, mueq, theta):
    """Solve the parametric LQ problems of ``batch`` (a handle with nth > 0) at ``theta`` [batch][nth] on
    ``torch.cuda.current_stream()``: set_problem, backward and the parametric forward pass.  Returns ``(xs, us, vs, vsT,
    lam0, lams)`` in the solver's output layouts, differentiable with respect to ``theta`` in both modes and to any
    order.  The solution is affine in theta, z = z_0 + J theta, and J comes from the stored factors without a new
    factorisation: a vjp is one ``theta_adjoint`` launch (J^T zbar), a jvp one ``theta_tangent`` launch (J d), and under
    vmap (``jacrev``, ``jacfwd``, ``hessian``) all the cotangents or tangents of a level go to one launch.  ``jacfwd`` is
    the cheap direction: nth tangents.  When another call has refactored the handle since (its ``factor_epoch``
    moved), set_problem and backward are run again before a derivative.  ``mueq`` (a number or a [batch] tensor) is not
    differentiated, nor is the problem data: ``stage``, ``term``, ``G0`` and ``g0`` that require grad raise
    ``ValueError``, as do handles without parameters (plain, dense, parallel) and a tensor that is not a contiguous
    float64 CUDA tensor of the handle's shape, all before any library call.  vmap over ``theta`` or the data raises
    ``NotImplementedError``."""
    if not isinstance(batch, _gar.CudaRiccatiBatch):
        raise ValueError("lq_solve_theta: `batch` must be a CudaRiccatiBatch")
    if batch.nth == 0 or batch.dense or batch.legs:
        raise ValueError(_NO_THETA_HANDLE)
    _check_inputs(batch, dict(stage=stage, term=term, G0=G0, g0=g0))
    for name, t in dict(stage=stage, term=term, G0=G0, g0=g0).items():
        if t.requires_grad:
            raise ValueError("lq_solve_theta: %s requires grad; derivatives with respect to the data of a parametric "
                             "problem are not served, only with respect to theta" % name)
    shape = (batch.dims.batch, batch.nth)
    if (not isinstance(theta, torch.Tensor) or theta.dtype != torch.float64 or not theta.is_cuda
            or not theta.is_contiguous() or tuple(theta.shape) != shape):
        raise ValueError("lq_solve_theta: theta must be a contiguous float64 CUDA tensor of shape %s" % (shape,))
    return _LqSolveTheta.apply(_Theta(batch, mueq), stage, term, G0, g0, theta)
