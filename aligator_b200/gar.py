"""Python host side of the CUDA batched Riccati sweep: a ctypes binding of the C ABI
(include/aligator_b200/gar.h) plus classes that mirror the reference's operator
interface for this path -- ``gar::RiccatiSolverBase`` (gar/riccati-base.hpp:13-37) as
implemented by ``gar::ProximalRiccatiSolver`` (gar/proximal-riccati.hpp:12-47).

There is NO CPU fallback: loading fails loudly when the CUDA library has not been
built, and every call fails loudly without a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import numbers
import os

import numpy as np

from .lqr import LqrProblem, lqr_initialize_solution

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libaligator_b200_gar.so")

AB2_HOST, AB2_DEVICE = 0, 1
(OUT_FF, OUT_FB, OUT_VXX, OUT_VX, OUT_FFT, OUT_FBT, OUT_KKT0, OUT_XS, OUT_US, OUT_VS, OUT_VST,
 OUT_LBD0, OUT_LBDAS, OUT_FTH, OUT_VXT, OUT_VTT, OUT_VT, OUT_KKT0FTH, OUT_THGRAD, OUT_THHESS) = range(20)

_dp = C.POINTER(C.c_double)


class GarDims(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("nx", "nu", "nc", "nct", "nc0", "horizon", "batch", "device")]


_LQ_PTRS = ("Jx", "Ju", "slack", "Lxx", "Lxu", "Luu", "Lx", "Lu", "Hxx", "Hxu", "Huu", "cJx", "cJu", "Lv",
            "shifted", "lo", "hi", "Lxx_N", "Lx_N", "cJx_N", "Lv_N", "shifted_N", "loN", "hiN", "G0", "g0", "Hxx0")


class LqInputs(C.Structure):
    """``ab2_lq_inputs``: device pointers to the derivative buffers of updateLQSubproblem."""
    _fields_ = [(n, C.c_void_p) for n in _LQ_PTRS] + [("preg", C.c_double), ("mu_inv", C.c_double)]


_FDDP_KEYS = ("Jx", "Ju", "fs", "Lxx", "Lxu", "Luu", "Lx", "Lu", "Lxx_N", "Lx_N")


class FddpInputs(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _FDDP_KEYS] + [("preg", C.c_double)]


_LS_KEYS = ("xs", "us", "vs", "vsT", "lam0", "lams")


class LsIterate(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _LS_KEYS]


_GRAD_KEYS = ("stage", "term", "G0", "g0")


class LqGrad(C.Structure):
    """``ab2_lq_grad``: device outputs of ``ab2_gar_adjoint`` (NULL = not wanted)."""
    _fields_ = [(k, C.c_void_p) for k in _GRAD_KEYS]


class LqTangent(C.Structure):
    """``ab2_lq_tangent``: device tangent records of ``ab2_gar_tangent`` (NULL = zero), keyed like ``LqGrad``."""
    _fields_ = [(k, C.c_void_p) for k in _GRAD_KEYS]


_RHS_KEYS = ("q", "r", "d", "dN", "g0", "f")


class LqRhs(C.Structure):
    """``ab2_lq_rhs``: device right-hand sides of ``ab2_gar_resolve`` (NULL = zero), [nrhs][batch][...]."""
    _fields_ = [(k, C.c_void_p) for k in _RHS_KEYS]


_FCOT_KEYS = ("ff", "fb", "vxx", "vx", "fft", "fbt")


class FactorCotangent(C.Structure):
    """``ab2_factor_cotangent``: device cotangents of ``ab2_gar_factor_adjoint`` (NULL = zero), in ``ab2_gar_get``'s
    layouts."""
    _fields_ = [(k, C.c_void_p) for k in _FCOT_KEYS]


class FactorTangent(C.Structure):
    """``ab2_factor_tangent``: device outputs of ``ab2_gar_factor_tangent`` (NULL = not written), in ``ab2_gar_get``'s
    layouts."""
    _fields_ = [(k, C.c_void_p) for k in _FCOT_KEYS]


class LqRefineWork(C.Structure):
    """``ab2_lq_refine_work``: caller-owned scratch of ``ab2_gar_refine_many``, the residual in resolve's rhs layouts
    (q .. f) and the correction in the solution's layouts (xs .. lams)."""
    _fields_ = [(k, C.c_void_p) for k in _RHS_KEYS + _LS_KEYS]


_MULT_IN = ("xs", "lam0", "lams", "vs", "vsT", "prev_vs", "prev_vsT", "init_value", "xnext", "fs", "cval", "cval_N",
            "lo", "hi", "loN", "hiN")
_MULT_OUT = ("slack", "lam0_plus", "lams_plus", "vs_plus", "vsT_plus", "shifted", "shifted_N", "Lv", "Lv_N")


class MultInputs(C.Structure):
    """``ab2_mult_inputs``: device pointers of computeMultipliers' inputs, then mu, mu_dyn."""
    _fields_ = [(k, C.c_void_p) for k in _MULT_IN] + [("mu", C.c_double), ("mu_dyn", C.c_double)]


class MultOutputs(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _MULT_OUT]


_LAG_IN = ("lx", "lu", "lx_N", "Jx", "Ju", "cJx", "cJu", "cJx_N", "G0", "lam0", "lams", "vs", "vsT")
_LAG_OUT = ("Lx", "Lx_N", "Lu", "Lxs", "Lus")


class LagInputs(C.Structure):
    """``ab2_lag_inputs``: device pointers of LagrangianDerivatives::compute's inputs."""
    _fields_ = [(k, C.c_void_p) for k in _LAG_IN] + [("force_initial_condition", C.c_int)]


class LagOutputs(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _LAG_OUT]


def _fill(struct, keys, arrays):
    for k in keys:
        a = arrays.get(k)
        setattr(struct, k, None if a is None else _ptr(a).value)
    return struct


class GarTuning(C.Structure):
    _fields_ = [("variant", C.c_int), ("stagger_ns", C.c_int), ("ctas_per_sm", C.c_int)]


class GarError(RuntimeError):
    pass


_lib = None
# the calls ab2_gar_<name>(h, double mueq, ...) whose twin ab2_gar_<name>_v takes (mueq array, memspace) in its place
_MU_TWINS = ("backward", "sweep", "adjoint", "tangent", "resolve", "adjoint_many", "tangent_many", "refine",
             "refine_many", "factor_adjoint", "factor_tangent")


def lib():
    """The C-ABI library; raises if it has not been built (no silent fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GarError("%s not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback for this path)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.ab2_gar_last_error.restype = C.c_char_p
        L.ab2_gar_version.restype = C.c_char_p
        L.ab2_gar_stage_record_doubles.restype = C.c_size_t
        L.ab2_gar_term_record_doubles.restype = C.c_size_t
        L.ab2_gar_output_doubles.restype = C.c_size_t
        L.ab2_gar_output_doubles.argtypes = [C.c_void_p, C.c_int]
        L.ab2_gar_launch_count.restype = C.c_long
        L.ab2_gar_launch_count.argtypes = [C.c_void_p]
        L.ab2_gar_create.argtypes = [C.POINTER(GarDims), C.POINTER(C.c_void_p)]
        L.ab2_gar_destroy.argtypes = [C.c_void_p]
        L.ab2_gar_set_tuning.argtypes = [C.c_void_p, C.POINTER(GarTuning)]
        L.ab2_gar_set_problem.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_int, C.c_void_p]
        L.ab2_gar_backward.argtypes = [C.c_void_p, C.c_double, C.c_void_p]
        L.ab2_gar_forward.argtypes = [C.c_void_p, C.c_void_p]
        L.ab2_gar_sweep.argtypes = [C.c_void_p, C.c_double, C.c_void_p]
        L.ab2_gar_create_parametric.argtypes = [C.POINTER(GarDims), C.c_int, C.POINTER(C.c_void_p)]
        L.ab2_gar_create_parallel.argtypes = [C.POINTER(GarDims), C.c_int, C.POINTER(C.c_void_p)]
        L.ab2_gar_create_dense.argtypes = [C.POINTER(GarDims), C.POINTER(C.c_void_p)]
        L.ab2_gar_collapse_feedback.argtypes = [C.c_void_p, C.c_void_p]
        L.ab2_gar_stage_record_doubles_th.restype = C.c_size_t
        L.ab2_gar_term_record_doubles_th.restype = C.c_size_t
        L.ab2_gar_forward_theta.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_sweep_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_double, C.c_int, C.POINTER(C.c_int),
                                         C.POINTER(C.c_void_p), C.c_int, C.c_void_p]
        L.ab2_gar_sweep_host_sym.argtypes = L.ab2_gar_sweep_host.argtypes
        L.ab2_gar_sweep_host_v.argtypes = L.ab2_gar_sweep_host.argtypes[:5] + [C.c_void_p] + L.ab2_gar_sweep_host.argtypes[6:]
        L.ab2_gar_sweep_host_sym_v.argtypes = L.ab2_gar_sweep_host_v.argtypes
        L.ab2_gar_stage_record_doubles_sym.restype = C.c_size_t
        L.ab2_gar_stage_record_doubles_sym.argtypes = [C.c_int, C.c_int, C.c_int]
        L.ab2_gar_pack_stage_sym.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_long]
        L.ab2_gar_get.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_get_range.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_assemble.argtypes = [C.c_void_p, C.POINTER(LqInputs), C.c_void_p]
        L.ab2_gar_assemble_v.argtypes = [C.c_void_p, C.POINTER(LqInputs), C.c_void_p, C.c_void_p, C.c_void_p]
        L.ab2_gar_get_problem.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_problem_ptr.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L.ab2_gar_kkt_error.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_kkt_error_v.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_get_gains.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_first_step_policy.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.ab2_gar_device_ptr.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L.ab2_gar_status.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_pivot_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_fddp_backward_pass.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ab2_fddp_backward_pass_v.argtypes = [C.c_void_p] * 6
        L.ab2_gar_linear_step.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ab2_gar_linear_step_v.argtypes = [C.c_void_p] * 5
        L.ab2_gar_directional_derivative.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_al_value.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_al_value_v.argtypes = [C.c_void_p] * 6 + [C.c_int, C.c_void_p]
        L.ab2_gar_adjoint.argtypes = [C.c_void_p, C.c_double, C.POINTER(LsIterate), C.POINTER(LsIterate),
                                      C.POINTER(LqGrad), C.c_void_p]
        L.ab2_gar_tangent.argtypes = [C.c_void_p, C.c_double, C.POINTER(LsIterate), C.POINTER(LqTangent), C.c_void_p]
        L.ab2_gar_resolve.argtypes = [C.c_void_p, C.c_double, C.c_int, C.POINTER(LqRhs), C.POINTER(LsIterate),
                                      C.c_void_p]
        L.ab2_gar_factor_epoch.argtypes = [C.c_void_p, C.POINTER(C.c_longlong)]
        L.ab2_gar_theta_tangent.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.POINTER(LsIterate), C.c_void_p]
        L.ab2_gar_theta_adjoint.argtypes = [C.c_void_p, C.c_int, C.POINTER(LsIterate), C.c_void_p, C.c_void_p]
        L.ab2_gar_adjoint_many.argtypes = [C.c_void_p, C.c_double, C.c_int, C.POINTER(LsIterate), C.POINTER(LsIterate),
                                           C.POINTER(LsIterate), C.POINTER(LqGrad), C.c_void_p]
        L.ab2_gar_tangent_many.argtypes = [C.c_void_p, C.c_double, C.c_int, C.POINTER(LsIterate), C.POINTER(LqTangent),
                                           C.POINTER(LsIterate), C.POINTER(LsIterate), C.c_void_p]
        L.ab2_gar_rho_many.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(LqTangent), C.POINTER(LsIterate), C.c_int,
                                       C.POINTER(LqTangent), C.POINTER(LsIterate), C.c_int, C.POINTER(LsIterate),
                                       C.POINTER(LsIterate), C.c_void_p]
        L.ab2_gar_grad_many.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(LsIterate), C.POINTER(LsIterate), C.c_int,
                                        C.POINTER(LsIterate), C.POINTER(LsIterate), C.c_int, C.POINTER(LqGrad),
                                        C.c_void_p]
        L.ab2_gar_refine.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
        L.ab2_gar_refine_many.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_int, C.POINTER(LqRhs),
                                          C.POINTER(LsIterate), C.POINTER(LqRefineWork), C.c_void_p, C.c_void_p]
        L.ab2_gar_factor_adjoint.argtypes = [C.c_void_p, C.c_double, C.POINTER(FactorCotangent), C.POINTER(LqGrad),
                                             C.c_void_p]
        L.ab2_gar_factor_tangent.argtypes = [C.c_void_p, C.c_double, C.POINTER(LqTangent), C.POINTER(FactorTangent),
                                             C.c_void_p]
        L.ab2_gar_multipliers.argtypes = [C.c_void_p, C.POINTER(MultInputs), C.POINTER(MultOutputs), C.c_void_p, C.c_int,
                                          C.c_void_p]
        L.ab2_gar_multipliers_v.argtypes = [C.c_void_p, C.POINTER(MultInputs), C.c_void_p, C.c_void_p,
                                            C.POINTER(MultOutputs), C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_lagrangian_gradient.argtypes = [C.c_void_p, C.POINTER(LagInputs), C.POINTER(LagOutputs), C.c_void_p]
        L.ab2_gar_criterion.argtypes = [C.c_void_p] + [C.c_void_p] * 7 + [C.c_int, C.c_void_p]
        L.ab2_gar_peer_gather_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.ab2_gar_peer_gather_connect.argtypes = [C.c_void_p, C.c_void_p]
        L.ab2_gar_policy_allgather.argtypes = [C.c_void_p, C.c_void_p]
        L.ab2_gar_policy_allgather_wait.argtypes = [C.c_void_p, C.c_void_p]
        L.ab2_gar_peer_gather_buffer.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.ab2_gar_cycle_append.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.ab2_gar_synchronize.argtypes = [C.c_void_p, C.c_void_p]
        L.ab2_gar_kernel_info.argtypes = [C.c_void_p] + [C.POINTER(C.c_int)] * 5
        for name in _MU_TWINS:  # ab2_gar_<name>_v(h, mueq array, memspace, ...): the scalar mueq's place
            getattr(L, "ab2_gar_%s_v" % name).argtypes = ([C.c_void_p, C.c_void_p, C.c_int]
                                                          + getattr(L, "ab2_gar_" + name).argtypes[2:])
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise GarError("aligator_b200 gar error %d: %s" % (rc, lib().ab2_gar_last_error().decode()))


def stage_record_doubles(nx, nu, nc):
    return int(lib().ab2_gar_stage_record_doubles(nx, nu, nc))


def term_record_doubles(nx, nct):
    return int(lib().ab2_gar_term_record_doubles(nx, nct))


def supported(nx, nu, nc, nc0):
    """0: not served; 1: compile-time shape (warp per instance); 2: run-time shape (CTA per
    instance, csrc/riccati_block.cuh)."""
    return int(lib().ab2_gar_supported(nx, nu, nc, nc0))


def _ptr(a):
    """Raw address of a numpy array / torch tensor / int."""
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    if isinstance(a, np.ndarray):
        return C.c_void_p(a.ctypes.data)
    if hasattr(a, "data_ptr"):
        return C.c_void_p(a.data_ptr())
    raise TypeError(type(a))


class CudaRiccatiBatch:
    """Thin owner of an ``ab2_gar_solver`` handle: `batch` independent LQ problems of
    identical dimensions (stage knots (nx,nu,nc), terminal knot (nx,0,nct))."""

    def __init__(self, nx, nu, nc, nct, nc0, horizon, batch, device=0, variant=-1, stagger_ns=0,
                 ctas_per_sm=0, nth=0, legs=0, dense=False):
        """``legs >= 2``: the parallel-in-time solver (``ab2_gar_create_parallel`` =
        gar::ParallelRiccatiSolver): plain records, value-function parameters nth = nx."""
        self.dims = GarDims(nx, nu, nc, nct, nc0, horizon, batch, device)
        self.legs = int(legs)
        self.dense = bool(dense)
        self.nth = int(nx) if self.legs else int(nth)
        self.h = C.c_void_p()
        if self.dense:  # gar::RiccatiSolverDense (ab2_gar_create_dense)
            _check(lib().ab2_gar_create_dense(C.byref(self.dims), C.byref(self.h)))
        elif self.legs:
            _check(lib().ab2_gar_create_parallel(C.byref(self.dims), self.legs, C.byref(self.h)))
        else:
            _check(lib().ab2_gar_create_parametric(C.byref(self.dims), self.nth, C.byref(self.h)))
        if variant >= 0 or stagger_ns or ctas_per_sm:
            _check(lib().ab2_gar_set_tuning(self.h, C.byref(GarTuning(variant, stagger_ns, ctas_per_sm))))
        rec_nth = 0 if self.legs else self.nth
        self.srec = int(lib().ab2_gar_stage_record_doubles_th(nx, nu, nc, rec_nth))
        self.trec = int(lib().ab2_gar_term_record_doubles_th(nx, nct, rec_nth))
        self._keep = {}  # call name -> the arguments of its last call, alive while the device may still read them
        self._keep_v = {}

    # ---- per-instance scalars (the *_v twins of the C ABI) ----------------------
    def _per_instance(self, v, name):
        """None when `v` is a Python number (the scalar call), else `v` itself after checking that it is a 1-D
        float64 numpy array or torch tensor of length batch (ValueError otherwise)."""
        if isinstance(v, numbers.Real) or getattr(v, "ndim", None) == 0:  # numbers, numpy scalars, 0-d arrays
            return None
        B = self.dims.batch
        if isinstance(v, np.ndarray):
            ok = v.dtype == np.float64 and v.ndim == 1 and v.shape[0] == B
        elif hasattr(v, "data_ptr") and hasattr(v, "is_cuda"):
            import torch
            ok = v.dtype == torch.float64 and v.dim() == 1 and v.shape[0] == B
        else:
            ok = False
        if not ok:
            raise ValueError("%s: expected a number or a 1-D float64 array / tensor of length batch = %d" % (name, B))
        return v

    def _host_array(self, v, name):
        """A checked per-instance array as contiguous host memory, kept alive by the handle."""
        if not isinstance(v, np.ndarray):
            v = v.detach().cpu().numpy()
        v = np.ascontiguousarray(v)
        self._keep_v[name] = v
        return v

    def _device_array(self, v, name, stream):
        """A checked per-instance array as contiguous device memory: CUDA tensors as they are, host arrays uploaded.
        Kept alive by the handle until the next call that passes `name`; with a non-default stream the allocator
        is told that the stream uses it."""
        import torch
        if not (isinstance(v, torch.Tensor) and v.is_cuda):
            host = v if isinstance(v, np.ndarray) else v.detach().numpy()
            v = torch.from_numpy(np.ascontiguousarray(host)).to("cuda:%d" % self.dims.device)
            if stream:
                v.record_stream(torch.cuda.ExternalStream(stream))
        else:
            v = v.contiguous()
        self._keep_v[name] = v
        return v

    def _device_pair(self, a, b, names, stream):
        """Two per-instance scalars of one call: None when both are numbers, else both as device arrays (a number
        given beside an array applies to every instance)."""
        va, vb = self._per_instance(a, names[0]), self._per_instance(b, names[1])
        if va is None and vb is None:
            return None
        B = self.dims.batch
        va = np.full(B, float(a)) if va is None else va
        vb = np.full(B, float(b)) if vb is None else vb
        return self._device_array(va, names[0], stream), self._device_array(vb, names[1], stream)

    def _mueq_arg(self, mueq, stream):
        """(pointer, memspace) of a per-instance mu for backward_v / sweep_v, or None for a number."""
        v = self._per_instance(mueq, "mueq")
        if v is None:
            return None
        if hasattr(v, "is_cuda") and v.is_cuda:
            return _ptr(self._device_array(v, "mueq", stream)), AB2_DEVICE
        return _ptr(self._host_array(v, "mueq")), AB2_HOST

    def _mu_call(self, name, mueq, stream, keep, *args):
        """``ab2_gar_<name>(h, mueq, *args, stream)`` for a number ``mueq``, else ``ab2_gar_<name>_v(h, array,
        memspace, *args, stream)``.  ``keep``: the arrays behind ``args``, kept alive until the next call of ``name``."""
        v = self._mueq_arg(mueq, stream)
        if keep is not None:
            self._keep[name] = keep
        if v is None:
            _check(getattr(lib(), "ab2_gar_" + name)(self.h, float(mueq), *args, C.c_void_p(stream)))
        else:
            _check(getattr(lib(), "ab2_gar_%s_v" % name)(self.h, v[0], v[1], *args, C.c_void_p(stream)))

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            lib().ab2_gar_destroy(self.h)
            self.h = C.c_void_p()

    __del__ = close

    # ---- problem data -------------------------------------------------------
    def set_problem(self, stage=None, term=None, G0=None, g0=None, memspace=AB2_HOST, stream=0):
        """stage [batch][N][srec], term [batch][trec], G0 [batch][nc0*nx] (col-major
        blocks), g0 [batch][nc0]; host numpy arrays or device pointers/tensors."""
        if memspace == AB2_HOST:
            conv = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)
            stage, term, G0, g0 = conv(stage), conv(term), conv(G0), conv(g0)
            d = self.dims
            if stage is not None:
                assert stage.size == d.batch * d.horizon * self.srec, "stage size"
            if term is not None:
                assert term.size == d.batch * self.trec, "term size"
        self._keep["set_problem"] = (stage, term, G0, g0)
        _check(lib().ab2_gar_set_problem(self.h, _ptr(stage), _ptr(term), _ptr(G0), _ptr(g0),
                                         memspace, C.c_void_p(stream)))

    # ---- the hot calls ------------------------------------------------------
    def backward(self, mueq, stream=0):
        """``mueq``: a number, or a [batch] float64 array / tensor of per-instance values (``ab2_gar_backward_v``;
        CUDA tensors are read on the device, host arrays are staged by the library)."""
        self._mu_call("backward", mueq, stream, None)

    def forward(self, stream=0, theta=None):
        """forward(); with ``theta`` ([batch][nth]) the parametric rollout.  A CUDA tensor is read on the device,
        stream-ordered (no synchronisation); anything else is copied from the host and the call synchronises."""
        if theta is None:
            _check(lib().ab2_gar_forward(self.h, C.c_void_p(stream)))
        elif hasattr(theta, "is_cuda") and theta.is_cuda:
            import torch
            if theta.dtype != torch.float64 or theta.numel() != self.dims.batch * self.nth:
                raise ValueError("theta: expected %d float64 values ([batch][nth])" % (self.dims.batch * self.nth))
            th = theta.contiguous()
            self._keep["forward"] = th
            _check(lib().ab2_gar_forward_theta(self.h, _ptr(th), AB2_DEVICE, C.c_void_p(stream)))
        else:
            th = np.ascontiguousarray(theta, dtype=np.float64)
            assert th.size == self.dims.batch * self.nth
            self._keep["forward"] = th
            _check(lib().ab2_gar_forward_theta(self.h, _ptr(th), AB2_HOST, C.c_void_p(stream)))
            self.synchronize(stream)

    def collapse_feedback(self, stream=0):
        _check(lib().ab2_gar_collapse_feedback(self.h, C.c_void_p(stream)))

    def sweep(self, mueq, stream=0):
        """``mueq``: a number or a [batch] array / tensor (``ab2_gar_sweep_v``), as for ``backward``."""
        self._mu_call("sweep", mueq, stream, None)

    def synchronize(self, stream=0):
        _check(lib().ab2_gar_synchronize(self.h, C.c_void_p(stream)))

    def _sweep_host(self, name, stage, term, G0, g0, mueq, outputs, nchunks, stream):
        """``ab2_gar_<name>`` or, for a per-instance ``mueq``, ``ab2_gar_<name>_v`` (the array staged from the host)."""
        v = self._per_instance(mueq, "mueq")
        whats = (C.c_int * len(outputs))(*outputs.keys())
        dsts = (C.c_void_p * len(outputs))(*[_ptr(a).value for a in outputs.values()])
        self._keep["sweep_host"] = (stage, term, G0, g0, outputs)
        if v is None:
            f, mu = getattr(lib(), "ab2_gar_" + name), C.c_double(mueq)
        else:
            f, mu = getattr(lib(), "ab2_gar_%s_v" % name), _ptr(self._host_array(v, "mueq"))
        _check(f(self.h, _ptr(stage), _ptr(term), _ptr(G0), _ptr(g0), mu, int(nchunks), whats, dsts, len(outputs),
                 C.c_void_p(stream)))

    def sweep_host(self, stage, term, G0, g0, mueq, outputs, nchunks=0, stream=0):
        """Upload + sweep + download in one pipelined call (``ab2_gar_sweep_host``): the batch
        travels in slices on internal streams so uploads, sweeps and downloads overlap.
        ``outputs``: {OUT_*: host array of the full output size}; pinned arrays make the
        copies asynchronous.  Asynchronous w.r.t. the host: call ``synchronize(stream)``.  ``mueq``: a number or a
        [batch] array / tensor of per-instance values (``ab2_gar_sweep_host_v``)."""
        self._sweep_host("sweep_host", stage, term, G0, g0, mueq, outputs, nchunks, stream)

    def sweep_host_sym(self, stage_sym, term, G0, g0, mueq, outputs, nchunks=0, stream=0):
        """``sweep_host`` with the symmetric blocks Q, R of every stage knot sent as lower triangles
        (``ab2_gar_sweep_host_sym``; records made by ``pack_stage_sym``): fewer bytes over PCIe.  ``mueq``: a number
        or a [batch] array / tensor (``ab2_gar_sweep_host_sym_v``)."""
        self._sweep_host("sweep_host_sym", stage_sym, term, G0, g0, mueq, outputs, nchunks, stream)

    def pack_stage_sym(self, stage, out=None):
        """Full stage records [batch][N][srec] (host) -> triangle-packed records (``ab2_gar_pack_stage_sym``)."""
        d = self.dims
        n = int(lib().ab2_gar_stage_record_doubles_sym(d.nx, d.nu, d.nc))
        nrec = d.batch * d.horizon
        if out is None:
            out = np.empty(max(nrec * n, 1), dtype=np.float64)
        _check(lib().ab2_gar_pack_stage_sym(d.nx, d.nu, d.nc, _ptr(stage), _ptr(out), C.c_long(nrec)))
        return out

    # ---- results ------------------------------------------------------------
    def out_shape(self, what):
        d = self.dims
        nr = d.nu + d.nc + d.nx + (d.nx if getattr(self, "dense", False) else 0)
        return {
            OUT_FF: (d.batch, d.horizon, nr), OUT_FB: (d.batch, d.horizon, nr, d.nx),
            OUT_VXX: (d.batch, d.horizon + 1, d.nx, d.nx), OUT_VX: (d.batch, d.horizon + 1, d.nx),
            OUT_FFT: (d.batch, d.nct), OUT_FBT: (d.batch, d.nct, d.nx),
            OUT_KKT0: (d.batch, d.nx + d.nc0), OUT_XS: (d.batch, d.horizon + 1, d.nx),
            OUT_US: (d.batch, d.horizon, d.nu), OUT_VS: (d.batch, d.horizon, d.nc),
            OUT_VST: (d.batch, d.nct), OUT_LBD0: (d.batch, d.nc0),
            OUT_LBDAS: (d.batch, d.horizon, d.nx),
            OUT_FTH: (d.batch, d.horizon, nr, self.nth), OUT_VXT: (d.batch, d.horizon + 1, self.nth, d.nx),
            OUT_VTT: (d.batch, d.horizon + 1, self.nth, self.nth), OUT_VT: (d.batch, d.horizon + 1, self.nth),
            OUT_KKT0FTH: (d.batch, d.nx + d.nc0, self.nth), OUT_THGRAD: (d.batch, self.nth),
            OUT_THHESS: (d.batch, self.nth, self.nth)}[what]

    def get(self, what, out=None, stream=0, sync=True):
        """Copy an output array to the host.  VXX blocks are column-major in memory; the
        returned array is indexed [b, t, i, j]."""
        shape = self.out_shape(what)
        n = int(np.prod(shape))
        assert n == lib().ab2_gar_output_doubles(self.h, what)
        buf = out if out is not None else np.empty(max(n, 1), dtype=np.float64)
        if n:
            _check(lib().ab2_gar_get(self.h, what, _ptr(buf), AB2_HOST, C.c_void_p(stream)))
            if sync:
                self.synchronize(stream)
        a = buf[:n].reshape(shape)
        if what in (OUT_VXX, OUT_VXT, OUT_VTT):  # column-major blocks -> [b, t, i, j]
            a = a.transpose(0, 1, 3, 2)
        elif what == OUT_THHESS:
            a = a.transpose(0, 2, 1)
        return a

    def get_into(self, what, dst, memspace, stream=0):
        _check(lib().ab2_gar_get(self.h, what, _ptr(dst), memspace, C.c_void_p(stream)))

    def get_range_into(self, what, b0, nb, t0, nt, dst, memspace, stream=0):
        _check(lib().ab2_gar_get_range(self.h, what, b0, nb, t0, nt, _ptr(dst), memspace,
                                       C.c_void_p(stream)))

    def assemble(self, arrays, preg, mu_inv, stream=0):
        """updateLQSubproblem + computeProjectedJacobians on the device (``ab2_gar_assemble``).
        ``arrays``: {field of ab2_lq_inputs: device tensor / device address}; missing fields
        are NULL.  The assembled problem becomes the solver's current problem.  ``preg``, ``mu_inv``: numbers, or
        [batch] arrays / tensors of per-instance values (``ab2_gar_assemble_v``)."""
        inp = LqInputs()
        for n in _LQ_PTRS:
            a = arrays.get(n)
            setattr(inp, n, None if a is None else _ptr(a).value)
        v = self._device_pair(preg, mu_inv, ("preg", "mu_inv"), stream)
        self._keep["assemble"] = (arrays,)
        if v is None:
            inp.preg, inp.mu_inv = float(preg), float(mu_inv)
            _check(lib().ab2_gar_assemble(self.h, C.byref(inp), C.c_void_p(stream)))
        else:
            _check(lib().ab2_gar_assemble_v(self.h, C.byref(inp), _ptr(v[0]), _ptr(v[1]), C.c_void_p(stream)))

    def get_problem(self, what, stream=0):
        """Host copy of the current packed problem: what = 0 stage, 1 term, 2 G0, 3 g0."""
        d = self.dims
        n = [d.batch * d.horizon * self.srec, d.batch * self.trec, d.batch * d.nc0 * d.nx, d.batch * d.nc0][what]
        buf = np.empty(max(n, 1), dtype=np.float64)
        _check(lib().ab2_gar_get_problem(self.h, what, _ptr(buf), AB2_HOST, C.c_void_p(stream)))
        self.synchronize(stream)
        return buf[:n]

    def problem_device_ptrs(self):
        """Device addresses of the solver-owned packed problem (stage, term, G0, g0)."""
        out = []
        for w in range(4):
            p = C.c_void_p()
            _check(lib().ab2_gar_problem_ptr(self.h, w, C.byref(p)))
            out.append(p.value)
        return out

    def kkt_error(self, mueq, stream=0):
        """[batch][3] = (dynamics, constraint, stationarity) infinity norms of lqrComputeKktError
        (gar/utils.hxx:88-182) for the current problem and the last forward pass, computed on the device.
        ``mueq``: a number or a [batch] array / tensor (``ab2_gar_kkt_error_v``)."""
        v = self._per_instance(mueq, "mueq")
        out = np.empty((self.dims.batch, 3), dtype=np.float64)
        if v is None:
            _check(lib().ab2_gar_kkt_error(self.h, C.c_double(mueq), _ptr(out), AB2_HOST, C.c_void_p(stream)))
        else:
            _check(lib().ab2_gar_kkt_error_v(self.h, _ptr(self._device_array(v, "mueq", stream)), _ptr(out), AB2_HOST,
                                             C.c_void_p(stream)))
        self.synchronize(stream)
        return out

    def get_gains(self, stream=0):
        """[batch][N][nx+1][nu+nc+nx] view of the column-major gain blocks ``[ff | fb]``
        (results_.gains_ layout): ``g[b, t, 0]`` is the feedforward, ``g[b, t, 1 + j]`` column j."""
        d = self.dims
        nr = d.nu + d.nc + d.nx
        buf = np.empty(max(d.batch * d.horizon * nr * (d.nx + 1), 1), dtype=np.float64)
        _check(lib().ab2_gar_get_gains(self.h, _ptr(buf), AB2_HOST, C.c_void_p(stream)))
        self.synchronize(stream)
        return buf[:d.batch * d.horizon * nr * (d.nx + 1)].reshape(d.batch, d.horizon, d.nx + 1, nr)

    def first_step_policy_into(self, dst, stream=0):
        """[K_0 | k_0] of every instance -> device buffer dst [batch][nu][nx+1]."""
        _check(lib().ab2_gar_first_step_policy(self.h, _ptr(dst), C.c_void_p(stream)))

    def device_ptr(self, what):
        p = C.c_void_p()
        _check(lib().ab2_gar_device_ptr(self.h, what, C.byref(p)))
        return p.value

    def status(self, stream=0):
        st = np.empty(self.dims.batch, dtype=np.int32)
        _check(lib().ab2_gar_status(self.h, _ptr(st), AB2_HOST, C.c_void_p(stream)))
        self.synchronize(stream)
        return st

    # ---- multi-GPU: fused pack + all-gather of [K0 | k0] over NVLink peer memory ----
    def peer_gather_setup(self, dist, rank, world):
        """Allocate the receive buffer, exchange the CUDA IPC handles over `dist` (any backend)
        and map every peer's buffer.  All ranks: same batch."""
        import torch
        L = lib()
        h = (C.c_ubyte * 64)()
        # every rank takes part in both collectives whatever happens locally, and all ranks raise together:
        # a rank that cannot map its peers (no IPC / no peer access) must not leave the others waiting
        err = None
        if L.ab2_gar_peer_gather_init(self.h, int(world), int(rank), h) != 0:
            err = L.ab2_gar_last_error().decode()
        allh = [None] * world
        dist.all_gather_object(allh, (err, bytes(h)))
        if err is None and all(e is None for e, _ in allh):
            blob = (C.c_ubyte * (64 * world)).from_buffer_copy(b"".join(b for _, b in allh))
            if L.ab2_gar_peer_gather_connect(self.h, blob) != 0:
                err = L.ab2_gar_last_error().decode()
        errs = [None] * world
        dist.all_gather_object(errs, err)
        bad = [(r, e) for r, (e0, _) in enumerate(allh) for e in [e0 or errs[r]] if e]
        if bad:
            raise GarError("peer gather unavailable (rank %d: %s)" % bad[0])
        dist.barrier()
        torch.cuda.synchronize()

    def policy_allgather(self, stream=0):
        _check(lib().ab2_gar_policy_allgather(self.h, C.c_void_p(stream)))

    def policy_allgather_wait(self, stream=0):
        _check(lib().ab2_gar_policy_allgather_wait(self.h, C.c_void_p(stream)))

    def peer_gather_buffer(self):
        p, st = C.c_void_p(), C.c_long()
        _check(lib().ab2_gar_peer_gather_buffer(self.h, C.byref(p), C.byref(st)))
        return p.value, st.value

    # ---- line-search consumers (device tensors in, device tensors / host scalars out) ----
    def linear_step(self, alpha, current, trial, stream=0):
        """trial = current + alpha * step (tryLinearStep's vector part); `current` / `trial`: dicts with keys
        xs, us, vs, vsT, lam0, lams of device tensors laid out like the solver's outputs.  ``alpha``: a number or a
        [batch] array / tensor of per-instance step lengths (``ab2_gar_linear_step_v``)."""
        v = self._per_instance(alpha, "alpha")
        cur = LsIterate(*[_ptr(current.get(k)).value if current.get(k) is not None else None for k in _LS_KEYS])
        tr = LsIterate(*[_ptr(trial.get(k)).value if trial.get(k) is not None else None for k in _LS_KEYS])
        self._keep["linear_step"] = (current, trial)
        if v is None:
            _check(lib().ab2_gar_linear_step(self.h, C.c_double(alpha), C.byref(cur), C.byref(tr), C.c_void_p(stream)))
        else:
            _check(lib().ab2_gar_linear_step_v(self.h, _ptr(self._device_array(v, "alpha", stream)), C.byref(cur),
                                               C.byref(tr), C.c_void_p(stream)))

    def directional_derivative(self, Lxs, Lus, stream=0):
        out = np.empty(self.dims.batch, dtype=np.float64)
        _check(lib().ab2_gar_directional_derivative(self.h, _ptr(Lxs), _ptr(Lus), _ptr(out), AB2_HOST, C.c_void_p(stream)))
        self.synchronize(stream)
        return out

    def al_value(self, plus, cost, mudyn, mucstr, stream=0):
        """``mudyn``, ``mucstr``: numbers, or [batch] arrays / tensors of per-instance values (``ab2_gar_al_value_v``)."""
        v = self._device_pair(mudyn, mucstr, ("mudyn", "mucstr"), stream)
        it = LsIterate(*[_ptr(plus.get(k)).value if plus.get(k) is not None else None for k in _LS_KEYS])
        out = np.empty(self.dims.batch, dtype=np.float64)
        if v is None:
            _check(lib().ab2_gar_al_value(self.h, C.byref(it), _ptr(cost), C.c_double(mudyn), C.c_double(mucstr),
                                          _ptr(out), AB2_HOST, C.c_void_p(stream)))
        else:
            _check(lib().ab2_gar_al_value_v(self.h, C.byref(it), _ptr(cost), _ptr(v[0]), _ptr(v[1]), _ptr(out),
                                            AB2_HOST, C.c_void_p(stream)))
        self.synchronize(stream)
        return out

    # ---- gradients of the solution with respect to the problem data ----
    def adjoint(self, primal, cotangent, grad, mueq, stream=0):
        """Adjoint of the LQ solve (``ab2_gar_adjoint``): gradient records of a loss whose cotangents with respect to
        the solution are ``cotangent``.  ``primal``, ``cotangent``: dicts with keys xs, us, vs, vsT, lam0, lams of
        device tensors laid out like the solver's outputs (``primal``: the solution of the current problem at this
        mu; a cotangent key that is missing or None is zero).  ``grad``: dict with any of stage, term, G0, g0 of
        device tensors in the problem's layouts, overwritten.  ``mueq``: a number or a [batch] array / tensor
        (``ab2_gar_adjoint_v``).  Afterwards the handle's outputs are those of the adjoint solve."""
        pr = _fill(LsIterate(), _LS_KEYS, primal)
        ct = _fill(LsIterate(), _LS_KEYS, cotangent)
        gr = _fill(LqGrad(), _GRAD_KEYS, grad)
        self._mu_call("adjoint", mueq, stream, (primal, cotangent, grad), C.byref(pr), C.byref(ct), C.byref(gr))

    def tangent(self, primal, tangent, mueq, stream=0):
        """Forward mode of the LQ solve (``ab2_gar_tangent``): afterwards the handle's trajectory outputs (OUT_XS ..
        OUT_LBDAS) hold the derivative of the solution along the data tangent ``tangent``, a dict with any of stage,
        term, G0, g0 of device tensors in the problem's layouts (a key that is missing or None is zero).  ``primal``:
        dict with keys xs, us, vs, vsT, lam0, lams of device tensors or addresses laid out like the solver's outputs,
        the solution of the current problem at this mu; it may be the handle's own outputs (``device_ptr``).  The
        tangent of Q and R is taken through sym(.) = (. + .^T) / 2, as ``adjoint``'s gradient is.  ``mueq``: a number
        or a [batch] array / tensor (``ab2_gar_tangent_v``)."""
        pr = _fill(LsIterate(), _LS_KEYS, primal)
        dt = _fill(LqTangent(), _GRAD_KEYS, tangent)
        self._mu_call("tangent", mueq, stream, (primal, tangent), C.byref(pr), C.byref(dt))

    def resolve(self, rhs, out, mueq, stream=0):
        """Re-solve the last backward's LQ matrices for new vectors (``ab2_gar_resolve``): ``out`` receives
        z = -K^-1 h, the solution of the current problem with its vectors replaced by h.  ``rhs``: dict with any of
        q, r, d, dN, g0, f (a key that is missing or None is zero), ``out``: dict with keys xs, us, vs, vsT, lam0, lams;
        device tensors [nrhs][batch][...] in the layouts of the solution (q like xs, r like us, d like vs, dN like vsT,
        g0 like lam0, f like lams).  nrhs is read from ``out["xs"]``.  ``mueq``: the mu of the last backward, a number
        or a [batch] array / tensor (``ab2_gar_resolve_v``).  The handle's own outputs are not touched."""
        d = self.dims
        nrhs = out["xs"].numel() // (d.batch * (d.horizon + 1) * d.nx)
        rh = _fill(LqRhs(), _RHS_KEYS, rhs)
        ot = _fill(LsIterate(), _LS_KEYS, out)
        self._mu_call("resolve", mueq, stream, (rhs, out), int(nrhs), C.byref(rh), C.byref(ot))

    def theta_tangent(self, dtheta, out, stream=0):
        """J d for a parametric handle (``ab2_gar_theta_tangent``): the derivative of ``forward(theta=...)``'s
        solution along each direction d.  ``dtheta``: device tensor [nrhs][batch][nth]; ``out``: dict with keys xs, us,
        vs, vsT, lam0, lams of device tensors [nrhs][batch][...] in the solution's layouts, overwritten.  nrhs is read
        from ``dtheta``.  Reads only the last backward's factors; the handle's outputs are not touched."""
        d = self.dims
        nrhs = dtheta.numel() // (d.batch * self.nth)
        ot = _fill(LsIterate(), _LS_KEYS, out)
        self._keep["theta_tangent"] = (dtheta, out)
        _check(lib().ab2_gar_theta_tangent(self.h, int(nrhs), _ptr(dtheta), C.byref(ot), C.c_void_p(stream)))

    def theta_adjoint(self, cot, theta_bar, stream=0):
        """J^T zbar for a parametric handle (``ab2_gar_theta_adjoint``): the gradient with respect to theta of a loss
        whose cotangents with respect to the solution are ``cot``, a dict with any of xs, us, vs, vsT, lam0, lams of
        device tensors [nrhs][batch][...] (a key that is missing or None is zero).  ``theta_bar``: device tensor
        [nrhs][batch][nth], overwritten; nrhs is read from it.  Reads only the last backward's factors; the handle's
        outputs are not touched."""
        d = self.dims
        nrhs = theta_bar.numel() // (d.batch * self.nth)
        ct = _fill(LsIterate(), _LS_KEYS, cot)
        self._keep["theta_adjoint"] = (cot, theta_bar)
        _check(lib().ab2_gar_theta_adjoint(self.h, int(nrhs), C.byref(ct), _ptr(theta_bar), C.c_void_p(stream)))

    def adjoint_many(self, primal, cotangent, work, grad, mueq, stream=0):
        """Many cotangents on the last backward's factorisation (``ab2_gar_adjoint_many``): ``grad`` receives, for every
        cotangent j, the gradient records ``adjoint`` would give, and ``work`` receives y_j = -K^-1 zbar_j, the vector
        gradient in the solution's layouts.  ``primal``: dict with keys xs, us, vs, vsT, lam0, lams of device tensors
        [batch][...] (the solution of the current problem at this mu).  ``cotangent`` (a key that is missing or None is
        zero) and ``work``: dicts with the same keys of device tensors [nrhs][batch][...]; nrhs is read from
        ``work["xs"]``.  ``grad``: dict with any of stage, term, G0, g0 of device tensors [nrhs][batch][...] in the
        problem's layouts, overwritten (a missing key is not written).  ``mueq``: the mu of the last backward, a number
        or a [batch] array / tensor (``ab2_gar_adjoint_many_v``).  The handle's own outputs are not touched."""
        d = self.dims
        nrhs = work["xs"].numel() // (d.batch * (d.horizon + 1) * d.nx)
        pr = _fill(LsIterate(), _LS_KEYS, primal)
        ct = _fill(LsIterate(), _LS_KEYS, cotangent)
        wk = _fill(LsIterate(), _LS_KEYS, work)
        gr = _fill(LqGrad(), _GRAD_KEYS, grad)
        self._mu_call("adjoint_many", mueq, stream, (primal, cotangent, work, grad), int(nrhs), C.byref(pr), C.byref(ct),
                      C.byref(wk), C.byref(gr))

    def tangent_many(self, primal, tangent, work, out, mueq, stream=0):
        """Many tangents on the last backward's factorisation (``ab2_gar_tangent_many``): ``out`` receives, for every
        tangent j, the derivative zdot_j of the solution that ``tangent`` would give, and ``work`` the right-hand side
        rho_j = Kdot_j z + hdot_j in resolve's rhs layouts.  ``tangent``: dict with any of stage, term, G0, g0 of device
        tensors [nrhs][batch][...] in the problem's layouts (a key that is missing or None is zero).  ``primal``,
        ``work``, ``out``: dicts with keys xs, us, vs, vsT, lam0, lams of device tensors, [batch][...] for ``primal``
        and [nrhs][batch][...] for the others; nrhs is read from ``out["xs"]``.  ``mueq``: the mu of the last backward,
        a number or a [batch] array / tensor (``ab2_gar_tangent_many_v``).  The handle's own outputs are not
        touched."""
        d = self.dims
        nrhs = out["xs"].numel() // (d.batch * (d.horizon + 1) * d.nx)
        pr = _fill(LsIterate(), _LS_KEYS, primal)
        dt = _fill(LqTangent(), _GRAD_KEYS, tangent)
        wk = _fill(LsIterate(), _LS_KEYS, work)
        ot = _fill(LsIterate(), _LS_KEYS, out)
        self._mu_call("tangent_many", mueq, stream, (primal, tangent, work, out), int(nrhs), C.byref(pr), C.byref(dt),
                      C.byref(wk), C.byref(ot))

    def _each(self, v):
        """1 when the solution-layout dict ``v`` holds one vector per right-hand side ([nrhs][batch][...]), 0 when it is
        shared ([batch][...]), read from ``v["xs"]`` (at nrhs = 1 the two layouts are one: shared)."""
        d = self.dims
        return int(v["xs"].numel() != d.batch * (d.horizon + 1) * d.nx)

    def rho_many(self, dot, a, out, vectors=True, dot2=None, a2=None, e=None, stream=0):
        """``ab2_gar_rho_many``: ``out`` receives, for every right-hand side j, rho^(v)(dot_j; a_j) + rho_K(dot2_j; a2_j)
        + e_j in resolve's rhs layouts (rho^(v) = rho with the tangent's vector blocks when ``vectors``, rho_K without).
        ``dot``, ``dot2``: dicts with any of stage, term, G0, g0 of device tensors [nrhs][batch][...] in the problem's
        layouts (a key that is missing or None is zero; ``dot2`` None: no second term).  ``a``, ``a2``: dicts with keys
        xs, us, vs, vsT, lam0, lams of device tensors, [nrhs][batch][...] (one per right-hand side) or [batch][...]
        (shared), told apart by the size of ``xs``.  ``e`` (None: absent) and ``out``: the same keys, [nrhs][batch][...];
        nrhs is read from ``out["xs"]``.  Reads no factorisation and touches none of the handle's outputs."""
        d = self.dims
        nrhs = out["xs"].numel() // (d.batch * (d.horizon + 1) * d.nx)
        d1 = _fill(LqTangent(), _GRAD_KEYS, dot)
        a1 = _fill(LsIterate(), _LS_KEYS, a)
        d2 = None if dot2 is None else _fill(LqTangent(), _GRAD_KEYS, dot2)
        a2s = None if dot2 is None else _fill(LsIterate(), _LS_KEYS, a2)
        es = None if e is None else _fill(LsIterate(), _LS_KEYS, e)
        ot = _fill(LsIterate(), _LS_KEYS, out)
        self._keep["rho_many"] = (dot, a, dot2, a2, e, out)
        _check(lib().ab2_gar_rho_many(self.h, int(nrhs), int(bool(vectors)), C.byref(d1), C.byref(a1),
                                      self._each(a), None if d2 is None else C.byref(d2),
                                      None if a2s is None else C.byref(a2s),
                                      0 if dot2 is None else self._each(a2), None if es is None else C.byref(es),
                                      C.byref(ot), C.c_void_p(stream)))

    def grad_many(self, y, z, grad, vectors=True, y2=None, z2=None, stream=0):
        """``ab2_gar_grad_many``: ``grad`` receives, for every right-hand side j, Gr^(v)(y_j; z_j) + Gr_K(y2_j; z2_j):
        adjoint_many's gradient records for y and the primal z (Gr^(v) = Gr with the vector blocks when ``vectors``,
        Gr_K with them written 0).  ``y``, ``y2`` (None: no second pair): dicts with keys xs, us, vs, vsT, lam0, lams of
        device tensors [nrhs][batch][...]; nrhs is read from ``y["xs"]``.  ``z``, ``z2``: the same keys, [nrhs][batch][...]
        or [batch][...] (shared), told apart by the size of ``xs``.  ``grad``: dict with any of stage, term, G0, g0 of
        device tensors [nrhs][batch][...] in the problem's layouts, overwritten (a missing key is not written).  Reads no
        factorisation and touches none of the handle's outputs."""
        d = self.dims
        nrhs = y["xs"].numel() // (d.batch * (d.horizon + 1) * d.nx)
        ys, zs = _fill(LsIterate(), _LS_KEYS, y), _fill(LsIterate(), _LS_KEYS, z)
        y2s = None if y2 is None else _fill(LsIterate(), _LS_KEYS, y2)
        z2s = None if y2 is None else _fill(LsIterate(), _LS_KEYS, z2)
        gr = _fill(LqGrad(), _GRAD_KEYS, grad)
        self._keep["grad_many"] = (y, z, y2, z2, grad)
        _check(lib().ab2_gar_grad_many(self.h, int(nrhs), int(bool(vectors)), C.byref(ys), C.byref(zs),
                                       self._each(z), None if y2s is None else C.byref(y2s),
                                       None if z2s is None else C.byref(z2s),
                                       0 if y2 is None else self._each(z2), C.byref(gr), C.c_void_p(stream)))

    def refine(self, mueq, steps=1, norms=False, stream=0):
        """Iterative refinement of the handle's own trajectory outputs (OUT_XS .. OUT_LBDAS) against the current
        problem (``ab2_gar_refine``): ``steps`` times r = K z + h, z += resolve(r), on the last backward's
        factorisation.  Every other output is unchanged.  ``mueq``: the mu of the last backward, a number or a [batch]
        array / tensor (``ab2_gar_refine_v``).  With ``norms=True`` returns the [batch][steps + 1] infinity norms of the
        residual of the input iterate and of each refined iterate (numpy; the call then synchronises ``stream``)."""
        out = np.empty((self.dims.batch, steps + 1), dtype=np.float64) if norms else None
        self._mu_call("refine", mueq, stream, None, int(steps), _ptr(out))
        if out is not None:
            self.synchronize(stream)
        return out

    def refine_many(self, rhs, z, work, mueq, steps=1, norms=None, stream=0):
        """Iterative refinement of many resolve solutions at once (``ab2_gar_refine_many``): ``z`` (dict with keys xs,
        us, vs, vsT, lam0, lams of device tensors [nrhs][batch][...], e.g. ``resolve``'s ``out``) is refined in place
        towards -K^-1 h for the right-hand sides ``rhs`` (dict with any of q, r, d, dN, g0, f as for ``resolve``; a key
        that is missing or None is zero).  ``work``: dict with keys q, r, d, dN, g0, f (the last residual) and xs .. lams
        (the last correction) of device tensors [nrhs][batch][...].  nrhs is read from ``z["xs"]``.  ``mueq``: the mu of
        the last backward, a number or a [batch] array / tensor (``ab2_gar_refine_many_v``).  ``norms``: None (not
        written), True (returns a host [nrhs][batch][steps + 1] array after synchronising ``stream``) or a device
        tensor of that shape, written in stream order and returned."""
        d = self.dims
        nrhs = z["xs"].numel() // (d.batch * (d.horizon + 1) * d.nx)
        rh = _fill(LqRhs(), _RHS_KEYS, rhs)
        zz = _fill(LsIterate(), _LS_KEYS, z)
        wk = _fill(LqRefineWork(), _RHS_KEYS + _LS_KEYS, work)
        host = norms is True
        out = np.empty((nrhs, d.batch, steps + 1), dtype=np.float64) if host else norms
        self._mu_call("refine_many", mueq, stream, (rhs, z, work, out), int(nrhs), int(steps), C.byref(rh), C.byref(zz),
                      C.byref(wk), _ptr(out))
        if host:
            self.synchronize(stream)
        return out

    def factor_adjoint(self, cotangent, grad, mueq, stream=0):
        """Gradients of the factorisation (``ab2_gar_factor_adjoint``): ``grad`` receives the gradient records of a loss
        whose cotangents with respect to the last backward's outputs are ``cotangent``, a dict with any of ff, fb, vxx,
        vx, fft, fbt of device tensors laid out like ``get`` returns OUT_FF .. OUT_FBT (vxx as full blocks; a key that
        is missing or None is zero).  ``grad``: dict with any of stage, term, G0, g0 of device tensors in the problem's
        layouts, overwritten (G0 and g0 with zeros; a missing key is not written).  ``mueq``: the mu of the last
        backward, a number or a [batch] array / tensor (``ab2_gar_factor_adjoint_v``).  Needs a backward on the
        problem's own vectors since the last set_problem; the handle's outputs are not touched."""
        ct = _fill(FactorCotangent(), _FCOT_KEYS, cotangent)
        gr = _fill(LqGrad(), _GRAD_KEYS, grad)
        self._mu_call("factor_adjoint", mueq, stream, (cotangent, grad), C.byref(ct), C.byref(gr))

    def factor_tangent(self, dot, out, mueq, stream=0):
        """Forward mode of the factorisation (``ab2_gar_factor_tangent``): ``out`` receives the derivative of the last
        backward's outputs along the data tangent ``dot``, a dict with any of stage, term (G0 and g0 are ignored) of
        device tensors in the problem's layouts (a key that is missing or None is zero).  ``out``: dict with any of ff,
        fb, vxx, vx, fft, fbt of device tensors laid out like ``get`` returns OUT_FF .. OUT_FBT (vxx as full blocks),
        overwritten (a missing key is not written).  The tangent of Q and R is taken through sym(.) = (. + .^T) / 2.
        ``mueq``: the mu of the last backward, a number or a [batch] array / tensor (``ab2_gar_factor_tangent_v``).
        Needs a backward on the problem's own vectors since the last set_problem; the handle's outputs are not
        touched."""
        dt = _fill(LqTangent(), _GRAD_KEYS, dot)
        ot = _fill(FactorTangent(), _FCOT_KEYS, out)
        self._mu_call("factor_tangent", mueq, stream, (dot, out), C.byref(dt), C.byref(ot))

    def factor_epoch(self):
        """``ab2_gar_factor_epoch``: bumped by every call that rewrites the factorisation or the records."""
        e = C.c_longlong()
        _check(lib().ab2_gar_factor_epoch(self.h, C.byref(e)))
        return e.value

    # ---- multipliers, Lagrangian gradient, criterion (the rest of the inner iteration) ----
    def _scalars(self, call, out, stream):
        """Run `call(dst, memspace)` for a [batch][2] result: into the device tensor `out`, or to the host."""
        if out is not None:
            call(_ptr(out), AB2_DEVICE)
            return out
        host = np.empty((self.dims.batch, 2), dtype=np.float64)
        call(_ptr(host), AB2_HOST)
        self.synchronize(stream)
        return host

    def multipliers(self, inputs, outputs, mu, mu_dyn, out=None, stream=0):
        """computeMultipliers on the device (``ab2_gar_multipliers``).  ``inputs``: dict of device tensors keyed like
        ``ab2_mult_inputs`` (exactly one of xnext, fs); ``outputs``: dict of device tensors keyed like
        ``ab2_mult_outputs``.  Returns [batch][2] = [prim_infeas, finite (1.0 / 0.0)] as numpy, or writes it into the
        device tensor ``out`` and returns that.  ``mu``, ``mu_dyn``: numbers, or [batch] arrays / tensors of
        per-instance values (``ab2_gar_multipliers_v``)."""
        v = self._device_pair(mu, mu_dyn, ("mu", "mu_dyn"), stream)
        inp = _fill(MultInputs(), _MULT_IN, inputs)
        o = _fill(MultOutputs(), _MULT_OUT, outputs)
        self._keep["inner"] = (inputs, outputs)
        if v is None:
            inp.mu, inp.mu_dyn = float(mu), float(mu_dyn)
            return self._scalars(lambda dst, ms: _check(lib().ab2_gar_multipliers(
                self.h, C.byref(inp), C.byref(o), dst, ms, C.c_void_p(stream))), out, stream)
        return self._scalars(lambda dst, ms: _check(lib().ab2_gar_multipliers_v(
            self.h, C.byref(inp), _ptr(v[0]), _ptr(v[1]), C.byref(o), dst, ms, C.c_void_p(stream))), out, stream)

    def lagrangian_gradient(self, inputs, outputs, force_initial_condition=False, stream=0):
        """LagrangianDerivatives::compute on the device (``ab2_gar_lagrangian_gradient``).  ``inputs``: dict of
        device tensors keyed like ``ab2_lag_inputs``; ``outputs``: any of Lx, Lx_N, Lu (assemble layout) and Lxs,
        Lus (directional-derivative layout)."""
        inp = _fill(LagInputs(), _LAG_IN, inputs)
        inp.force_initial_condition = int(bool(force_initial_condition))
        o = _fill(LagOutputs(), _LAG_OUT, outputs)
        self._keep["inner"] = (inputs, outputs)
        _check(lib().ab2_gar_lagrangian_gradient(self.h, C.byref(inp), C.byref(o), C.c_void_p(stream)))

    def criterion(self, arrays, out=None, stream=0):
        """computeCriterion on the device (``ab2_gar_criterion``).  ``arrays``: dict of device tensors Lxs, Lus,
        init_value, slack, Lv, Lv_N.  Returns [batch][2] = [inner_criterion, dual_infeas] (numpy, or into ``out``)."""
        ptrs = [_ptr(arrays.get(k)) for k in ("Lxs", "Lus", "init_value", "slack", "Lv", "Lv_N")]
        self._keep["inner"] = (arrays,)
        return self._scalars(lambda dst, ms: _check(lib().ab2_gar_criterion(
            self.h, *ptrs, dst, ms, C.c_void_p(stream))), out, stream)

    def fddp_backward_pass(self, arrays, preg, Vx_out=None, Quuks_out=None, stream=0):
        """SolverFDDP::backwardPass on the device (``ab2_fddp_backward_pass``); ``arrays``: dict of device
        tensors Jx, Ju, fs, Lxx, Lxu, Luu, Lx, Lu, Lxx_N, Lx_N.  ``preg``: a number or a [batch] array / tensor of
        per-instance values (``ab2_fddp_backward_pass_v``)."""
        v = self._per_instance(preg, "preg")
        inp = FddpInputs(*[_ptr(arrays[k]).value for k in _FDDP_KEYS], 0.0 if v is not None else float(preg))
        self._keep["fddp_backward_pass"] = (arrays, Vx_out, Quuks_out)
        if v is None:
            _check(lib().ab2_fddp_backward_pass(self.h, C.byref(inp), _ptr(Vx_out), _ptr(Quuks_out),
                                                C.c_void_p(stream)))
        else:
            _check(lib().ab2_fddp_backward_pass_v(self.h, C.byref(inp), _ptr(self._device_array(v, "preg", stream)),
                                                  _ptr(Vx_out), _ptr(Quuks_out), C.c_void_p(stream)))

    def pivot_stats(self, stream=0):
        """(n_2x2, n_interchanges) per instance of the last backward pass (``ab2_gar_pivot_stats``)."""
        pv = np.empty(self.dims.batch, dtype=np.int32)
        _check(lib().ab2_gar_pivot_stats(self.h, _ptr(pv), AB2_HOST, C.c_void_p(stream)))
        self.synchronize(stream)
        self.kkt0_fast_path = ((pv >> 15) & 1).astype(bool)
        return pv & 0x7fff, (pv >> 16) & 0xffff

    def cycle_append(self, new_last, memspace=AB2_HOST, stream=0):
        if memspace == AB2_HOST:
            new_last = np.ascontiguousarray(new_last, dtype=np.float64)
            assert new_last.size == self.dims.batch * self.srec
        _check(lib().ab2_gar_cycle_append(self.h, _ptr(new_last), memspace, C.c_void_p(stream)))
        self.synchronize(stream)

    def launch_count(self):
        return int(lib().ab2_gar_launch_count(self.h))

    def kernel_info(self):
        v = [C.c_int() for _ in range(5)]
        _check(lib().ab2_gar_kernel_info(self.h, *[C.byref(x) for x in v]))
        d = dict(zip(("group_lanes", "smem_bytes_per_cta", "threads_per_cta", "grid",
                      "regs_per_thread"), [x.value for x in v]))
        d["ctas_per_sm"] = d["regs_per_thread"] >> 16
        d["regs_per_thread"] &= 0xffff
        return d


# ---------------------------------------------------------------------------
# packing of LqrProblem objects into the C-ABI layout
# ---------------------------------------------------------------------------
def _F(a):
    return np.asarray(a, dtype=np.float64).ravel(order="F")


def pack_stage_knot(k, srec):
    rec = np.concatenate([_F(k.A), _F(k.B), _F(k.f), _F(k.Q), _F(k.S), _F(k.R), _F(k.q), _F(k.r),
                          _F(k.C), _F(k.D), _F(k.d)])
    if k.nth:  # parametric blocks (gar/lqr-problem.hpp:66-71)
        rec = np.concatenate([rec, _F(k.Gx), _F(k.Gu), _F(k.Gv), _F(k.Gth), _F(k.gamma)])
    if rec.size < srec:
        rec = np.concatenate([rec, np.zeros(srec - rec.size)])
    return rec


def pack_term_knot(k):
    rec = np.concatenate([_F(k.Q), _F(k.q), _F(k.C), _F(k.d)])
    if k.nth:
        rec = np.concatenate([rec, _F(k.Gx), _F(k.Gv), _F(k.Gth), _F(k.gamma)])
    return rec


def _pad_terminal_controls(p):
    """A problem whose terminal knot has controls -> the equivalent problem in the library's layout
    (terminal nu = 0): knot N becomes a stage knot with A = B = f = 0 and a null terminal knot is
    appended.  The null knot's value function is zero, so the stage step at knot N reduces to the
    reference's terminal solve with controls (riccati-kernel.hxx:150-191): same K, k, Z, z, Vxx, vx;
    the co-state rows of knot N are exact zeros, the reference never writes them."""
    from .lqr import LqrKnot
    N = p.horizon
    kN = p.stages[N].copy()
    nx, nth = kN.nx, kN.nth
    kN.nx2 = nx
    kN.A, kN.B, kN.f = np.zeros((nx, nx), order="F"), np.zeros((nx, kN.nu), order="F"), np.zeros(nx)
    q = LqrProblem(list(p.stages[:N]) + [kN, LqrKnot(nx, 0, 0, nx, nth)], p.nc0)
    q.G0, q.g0 = p.G0, p.g0
    return q


def _pad_knot(k, nu, nc):
    """Stage knot with (k.nu, k.nc) <= (nu, nc) -> the equivalent knot of dims (nx, nu, nc): the extra
    controls are decoupled (R = I on their diagonal, zero S / B / r columns: their gains are exact
    zeros), the extra constraint rows are null (C = D = 0, d = 0: their multipliers are exact zeros).
    The KKT matrix is block diagonal with the caller's block first, so the factorisation of that block,
    interchanges included, is the reference's (tests/test_terminal_controls.py)."""
    from .lqr import LqrKnot
    if (k.nu, k.nc) == (nu, nc):
        return k
    if k.nu > nu or k.nc > nc:
        raise GarError("knot dims exceed the solver's")
    q = LqrKnot(k.nx, nu, nc, k.nx2, k.nth)
    q.Q[:], q.q[:], q.A[:], q.f[:] = k.Q, k.q, k.A, k.f
    q.S[:, :k.nu], q.B[:, :k.nu], q.r[:k.nu] = k.S, k.B, k.r
    q.R[:k.nu, :k.nu] = k.R
    q.R[range(k.nu, nu), range(k.nu, nu)] = 1.0
    q.C[:k.nc], q.D[:k.nc, :k.nu], q.d[:k.nc] = k.C, k.D, k.d
    if k.nth:
        q.Gth[:], q.Gx[:], q.gamma[:] = k.Gth, k.Gx, k.gamma
        q.Gu[:k.nu], q.Gv[:k.nc] = k.Gu, k.Gv
    return q


def _pad_stage_dims(p, nu, nc):
    q = LqrProblem([_pad_knot(k, nu, nc) for k in p.stages[:-1]] + [p.stages[-1]], p.nc0)
    q.G0, q.g0 = p.G0, p.g0
    return q


def pack_problems(problems):
    """Uniform-dims problems (terminal knot nu = 0, nth = 0) -> (stage, term, G0, g0)."""
    p0 = problems[0]
    N = p0.horizon
    k0 = p0.stages[0] if N > 0 else None
    kt = p0.stages[N]
    nx = kt.nx
    nu, nc = (k0.nu, k0.nc) if N > 0 else (1, 0)
    nth = p0.ntheta
    srec = int(lib().ab2_gar_stage_record_doubles_th(nx, nu, nc, nth))
    for p in problems:
        if p.horizon != N or p.nc0 != p0.nc0:
            raise GarError("all problems of a batch must share horizon and nc0")
        for t, s in enumerate(p.stages):
            want = (nx, nu, nc, nx, nth) if t < N else (nx, 0, kt.nc, s.nx2, nth)
            if s.dims != want:
                raise GarError("knot %d has dims %s, expected %s (uniform dims, terminal nu=0)"
                               % (t, s.dims, want))
    stage = np.empty((len(problems), N, srec))
    for b, p in enumerate(problems):
        for t in range(N):
            stage[b, t] = pack_stage_knot(p.stages[t], srec)
    term = np.stack([pack_term_knot(p.stages[N]) for p in problems])
    G0 = np.stack([_F(p.G0) for p in problems]) if p0.nc0 else np.zeros((len(problems), 0))
    g0 = np.stack([np.asarray(p.g0, dtype=np.float64) for p in problems]) if p0.nc0 \
        else np.zeros((len(problems), 0))
    return stage, term, G0, g0


class ProximalRiccatiSolver:
    """Mirror of ``gar::ProximalRiccatiSolver`` for ONE ``LqrProblem`` or a list of them
    (a batch).  Same call sequence as the reference:

        solver = ProximalRiccatiSolver(problem)      # proximal-riccati.hxx:13-31
        solver.backward(mueq)                        # riccati-base.hpp:19
        solver.forward(xs, us, vs, lbdas)            # riccati-base.hpp:21-24
        solver.getFeedforward(i); solver.getFeedback(i)   # riccati-base.hpp:33-34

    Like the reference it keeps a non-owning reference to the problem and re-reads it
    at every ``backward`` (the knots are rewritten in place between iterations).
    For a batch, ``forward`` takes lists of per-instance solution lists and the
    getters take ``(i, b)``.
    """

    def __init__(self, problem, device=0, variant=-1):
        self.problems = [problem] if isinstance(problem, LqrProblem) else list(problem)
        p0 = self.problems[0]
        N = p0.horizon
        kt = p0.stages[N]
        # A terminal knot WITH controls (terminalSolve's nu > 0 branch, riccati-kernel.hxx:150-173) is
        # solved as one more stage knot followed by a null terminal knot: the stage step from the zero
        # value function, with A = B = f = 0, is that branch exactly (see _pad_terminal_controls).
        self._term_controls = kt.nu != 0
        if self._term_controls:
            p0 = _pad_terminal_controls(p0)
            N = p0.horizon
            kt = p0.stages[N]
        # Stage knots of different (nu, nc) (gar/lqr-problem.hpp:49-118 lets every knot have its own) are
        # padded to the largest with decoupled controls / null constraint rows (_pad_knot).
        self._knot_dims = [(k.nu, k.nc) for k in p0.stages[:N]]
        self._ragged = len(set(self._knot_dims)) > 1
        if N > 0:
            nu, nc = max(d[0] for d in self._knot_dims), max(d[1] for d in self._knot_dims)
        else:
            nu, nc = 1, 0  # no stage knots: any instantiated shape serves
        self.nth = p0.ntheta  # parametric problems run the CTA-per-instance kernel
        self.nx, self.nu, self.nc, self.nct = kt.nx, nu, nc, kt.nc
        if N == 0:
            for cand in (2, 3, 1, 4, 6):
                if supported(self.nx, cand, 0, p0.nc0):
                    self.nu = cand
                    break
        self.batch = CudaRiccatiBatch(self.nx, self.nu, self.nc, self.nct, p0.nc0, N,
                                      len(self.problems), device, variant, nth=self.nth)
        self._single = isinstance(problem, LqrProblem)
        self._cache = {}

    # -- RiccatiSolverBase ---------------------------------------------------
    def backward(self, mueq):
        probs = [_pad_terminal_controls(p) for p in self.problems] if self._term_controls else self.problems
        if self._ragged:
            for p in probs:
                if [(k.nu, k.nc) for k in p.stages[:-1]] != self._knot_dims:
                    raise GarError("all problems of a batch must share the per-knot dims")
            probs = [_pad_stage_dims(p, self.nu, self.nc) for p in probs]
        stage, term, G0, g0 = pack_problems(probs)
        self.batch.set_problem(stage, term, G0, g0)
        self.batch.backward(mueq)
        self._cache = {}
        st = self.batch.status()
        if np.any(st & 1):
            # the reference throws here (riccati-kernel.hxx:239-241)
            raise GarError("Failed stage LDL factorization (instances %s)"
                           % np.nonzero(st & 1)[0][:8].tolist())
        return True

    def forward(self, xs, us, vs, lbdas, theta=None):
        if theta is not None:
            if self.nth == 0:
                raise GarError("theta given to a problem without parameters (nth = 0)")
            th = np.asarray(theta, dtype=np.float64).reshape(len(self.problems), self.nth)
            self.batch.forward(theta=th)
        else:
            self.batch.forward()
        B = self.batch
        N = B.dims.horizon
        X, U, V, VT = B.get(OUT_XS), B.get(OUT_US), B.get(OUT_VS), B.get(OUT_VST)
        L0, L = B.get(OUT_LBD0), B.get(OUT_LBDAS)
        sols = [(xs, us, vs, lbdas)] if self._single else list(zip(xs, us, vs, lbdas))
        if self._term_controls:  # internal horizon N = the caller's + 1; the null terminal knot is dropped
            for b, (x, u, v, l) in enumerate(sols):
                for t in range(N):
                    x[t][:] = X[b, t]
                    u[t][:] = U[b, t, :len(u[t])]
                    v[t][:] = V[b, t, :len(v[t])]
                    if t + 1 < N:
                        l[t + 1][:] = L[b, t]
                l[0][:] = L0[b]
            return True
        for b, (x, u, v, l) in enumerate(sols):
            for t in range(N + 1):
                x[t][:] = X[b, t]
            for t in range(N):
                u[t][:] = U[b, t, :len(u[t])]  # (ragged problems: the padding entries are dropped)
                v[t][:] = V[b, t, :len(v[t])]
                l[t + 1][:] = L[b, t]
            v[N][:] = VT[b]
            l[0][:] = L0[b]
        return True

    def collapseFeedback(self):
        """No-op for the serial solver (riccati-base.hpp:32)."""

    def _get(self, what):
        if what not in self._cache:
            self._cache[what] = self.batch.get(what)
        return self._cache[what]

    def _rows(self, i):
        """Rows of knot i's [k; z; a] blocks that belong to the caller's knot (all, unless padded)."""
        if not self._ragged:
            return slice(None)
        nu_i, nc_i = self._knot_dims[i]
        return np.r_[0:nu_i, self.nu:self.nu + nc_i, self.nu + self.nc:self.nu + self.nc + self.nx]

    def getFeedforward(self, i, b=0):
        """ff = [k; z; a] of knot i (length nu+nc+nx); the terminal knot's is [z]."""
        N = self.batch.dims.horizon
        return self._get(OUT_FFT)[b] if i == N else self._get(OUT_FF)[b, i][self._rows(i)]

    def getFeedback(self, i, b=0):
        """fb = [K; Z; Ahat] of knot i, (nu+nc+nx) x nx; the terminal knot's is [Z]."""
        N = self.batch.dims.horizon
        return self._get(OUT_FBT)[b] if i == N else self._get(OUT_FB)[b, i][self._rows(i)]

    def getFeedbackTheta(self, i, b=0):
        """fth = [Kth; Zth; Yth] of stage knot i, (nu+nc+nx) x nth (StageFactor::fth)."""
        return self._get(OUT_FTH)[b, i][self._rows(i)]

    def kkt0(self, b=0):
        """ff, fth of the initial stage and thGrad, thHess (proximal-riccati.hpp:40-43)."""
        return dict(ff=self._get(OUT_KKT0)[b], fth=self._get(OUT_KKT0FTH)[b],
                    thGrad=self._get(OUT_THGRAD)[b], thHess=self._get(OUT_THHESS)[b])

    def Vxx(self, i, b=0):
        return self._get(OUT_VXX)[b, i]

    def vx(self, i, b=0):
        return self._get(OUT_VX)[b, i]

    def kkt0_ff(self, b=0):
        return self._get(OUT_KKT0)[b]

    def cycleAppend(self, knot):
        """proximal-riccati.hxx:79-86; `knot`: an LqrKnot (same for the whole batch) or a
        list of one per instance.  The caller rotates its own problem objects, as
        SolverProxDDP::cycleProblem does (solver-proxddp.hxx:202-209)."""
        knots = [knot] * len(self.problems) if not isinstance(knot, (list, tuple)) else knot
        rec = np.stack([pack_stage_knot(k, self.batch.srec) for k in knots])
        self.batch.cycle_append(rec)
        self._cache = {}


class ParallelRiccatiSolver(ProximalRiccatiSolver):
    """Mirror of ``gar::ParallelRiccatiSolver`` (gar/parallel-solver.hpp:21-113) for ONE problem or a
    batch: ``ParallelRiccatiSolver(problem, num_threads)``.  The horizon is cut into ``num_threads``
    legs exactly like the reference (get_work, parallel-solver.hxx:23-28); on the device the legs of
    all instances run as the work items of one launch, followed by the condensed block-tridiagonal
    solve of every instance and the legs' rollouts.  Unlike the reference the caller's problem is
    NOT re-parameterised in place (the leg parameterisation is implicit on the device).  Raises
    like the reference for ``num_threads < 2`` (:42-46); ``forward`` ignores theta (:211)."""

    def __init__(self, problem, num_threads, device=0):
        self.problems = [problem] if isinstance(problem, LqrProblem) else list(problem)
        if num_threads < 2:
            raise GarError("numThreads (%d) should be greater than or equal to 2." % num_threads)
        p0 = self.problems[0]
        N = p0.horizon
        kt = p0.stages[N]
        if kt.nu != 0 or N < 1:
            raise GarError("the terminal knot must have nu = 0 and the horizon at least one stage knot")
        k0 = p0.stages[0]
        self.nx, self.nu, self.nc, self.nct = kt.nx, k0.nu, k0.nc, kt.nc
        self.nth = self.nx
        self.num_threads = int(num_threads)
        self._term_controls = False
        self._ragged = False
        self.batch = CudaRiccatiBatch(self.nx, self.nu, self.nc, self.nct, p0.nc0, N, len(self.problems),
                                      device, legs=self.num_threads)
        self._single = isinstance(problem, LqrProblem)
        self._cache = {}

    def getNumThreads(self):
        return self.num_threads

    def forward(self, xs, us, vs, lbdas, theta=None):
        return ProximalRiccatiSolver.forward(self, xs, us, vs, lbdas, None)  # theta ignored (:211)

    def collapseFeedback(self):
        """parallel-solver.hpp:41-51."""
        self.batch.collapse_feedback()
        self.batch.synchronize()
        self._cache = {}


def lqr_initialize_solution_batch(problems):
    sols = [lqr_initialize_solution(p) for p in problems]
    return tuple(list(z) for z in zip(*sols))
