"""ctypes binding of include/b200ldu.h (lib/libb200ldu.so) plus thin Python mirrors of the
reference's lduAddressing / lduMatrix / lduMatrix::solver interface.

PyTorch is used only for device memory (torch.Tensor on cuda) and streams; every compute
call goes through the C ABI.  There is no CPU fallback: a missing library or GPU raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200LDU_LIB: A/B experiments with differently compiled builds of the same library (tools/build_variant.sh)
LIB_PATH = os.path.abspath(os.environ.get("B200LDU_LIB") or os.path.join(_HERE, "lib", "libb200ldu.so"))


class B200LduError(RuntimeError):
    def __init__(self, rc, msg):
        super().__init__(f"b200ldu error {rc}: {msg}")
        self.rc = rc


class Controls(C.Structure):
    _fields_ = [
        ("tolerance", C.c_double), ("relTol", C.c_double),
        ("maxIter", C.c_int), ("minIter", C.c_int), ("nSweeps", C.c_int),
        ("omega", C.c_double), ("bicgstabRefQuirk", C.c_int),
        ("nCellsInCoarsestLevel", C.c_int), ("mergeLevels", C.c_int),
        ("nPreSweeps", C.c_int), ("preSweepsLevelMultiplier", C.c_int), ("maxPreSweeps", C.c_int),
        ("nPostSweeps", C.c_int), ("postSweepsLevelMultiplier", C.c_int), ("maxPostSweeps", C.c_int),
        ("nFinestSweeps", C.c_int), ("interpolateCorrection", C.c_int),
        ("scaleCorrection", C.c_int), ("directSolveCoarsest", C.c_int), ("checkEvery", C.c_int),
    ]


class Perf(C.Structure):
    _fields_ = [
        ("initialResidual", C.c_double), ("finalResidual", C.c_double), ("normFactor", C.c_double),
        ("nIterations", C.c_int), ("converged", C.c_int), ("singular", C.c_int),
        ("solverName", C.c_char * 64),
    ]

    def line(self, fieldName="p"):
        """The reference's solverPerformance::print line (SolverPerformance.C:96-123)."""
        nm = self.solverName.decode()
        if self.singular:
            return f"{nm}:  Solving for {fieldName}:  solution singularity"
        return (f"{nm}:  Solving for {fieldName}, Initial residual = {self.initialResidual:g}, "
                f"Final residual = {self.finalResidual:g}, No Iterations {self.nIterations}")


EXPORTS = [
    "b200ldu_last_error", "b200ldu_controls_default", "b200ldu_ctx_create", "b200ldu_ctx_destroy",
    "b200ldu_comm_unique_id", "b200ldu_comm_init", "b200ldu_comm_info", "b200ldu_ctx_set_stream", "b200ldu_ctx_sync",
    "b200ldu_addr_create", "b200ldu_addr_destroy", "b200ldu_addr_info", "b200ldu_addr_face_info",
    "b200ldu_addr_face_templates", "b200ldu_addr_perm",
    "b200ldu_matrix_create", "b200ldu_matrix_set", "b200ldu_matrix_destroy", "b200ldu_matrix_debug_trace",
    "b200ldu_matrix_debug_get",
    "b200ldu_amul", "b200ldu_tmul", "b200ldu_sumA", "b200ldu_residual", "b200ldu_H", "b200ldu_H1",
    "b200ldu_faceH", "b200ldu_precondition", "b200ldu_smooth",
    "b200ldu_vec_len", "b200ldu_to_banded", "b200ldu_from_banded", "b200ldu_amul_banded",
    "b200ldu_solve", "b200ldu_solve_host", "b200ldu_launch_count", "b200ldu_ctx_device_mem", "b200ldu_bench_op",
    "b200ldu_gamg_create", "b200ldu_gamg_destroy", "b200ldu_gamg_nlevels", "b200ldu_gamg_level_size",
    "b200ldu_gamg_restrict_addr", "b200ldu_gamg_debug_get", "b200ldu_gamg_debug_invert",
    "b200ldu_fv_boundary_set", "b200ldu_fv_surface_integrate", "b200ldu_fv_gauss_grad",
    "b200ldu_fv_laplacian_fill", "b200ldu_fv_convection_fill", "b200ldu_fv_interpolate_linear",
    "b200ldu_fv_add_boundary_diag", "b200ldu_fv_add_boundary_source", "b200ldu_fv_grad_linear",
    "b200ldu_fv_flux_linear",
    "b200ldu_fvm_add_boundary_diag", "b200ldu_fvm_add_boundary_source", "b200ldu_fvm_A", "b200ldu_fvm_H",
    "b200ldu_fvm_flux", "b200ldu_fvm_residual", "b200ldu_fvm_relax", "b200ldu_fvm_set_reference",
    "b200ldu_fvm_solve", "b200ldu_fv_patch_neighbour_field",
    "b200ldu_mules_limiter", "b200ldu_mules_limiter_corr", "b200ldu_ldu_row_sum", "b200ldu_ldu_add_assign", "b200ldu_ldu_scale", "b200ldu_fv_sngrad", "b200ldu_fv_limiter", "b200ldu_fv_limited_weights", "b200ldu_field_binary", "b200ldu_field_unary", "b200ldu_field_dot3", "b200ldu_field_symm_magsqr", "b200ldu_field_gather",
    "b200ldu_fvm_set_values", "b200ldu_wallfn_nutk", "b200ldu_wallfn_epsilon",
]

_lib = None
vp = C.c_void_p


def lib():
    """Load libb200ldu.so; raise loudly if it has not been built (no fallback path)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(nvcc, sm_90a). This package has no CPU or PyTorch fallback.")
    # torch bundles its own libnccl.so.2 (newer than the system one); load torch first so
    # both torch and this library resolve the same NCCL
    import torch  # noqa: F401
    L = C.CDLL(LIB_PATH)
    L.b200ldu_last_error.restype = C.c_char_p
    L.b200ldu_vec_len.restype = C.c_longlong
    L.b200ldu_vec_len.argtypes = [vp]
    L.b200ldu_launch_count.restype = C.c_longlong
    L.b200ldu_launch_count.argtypes = [vp]
    L.b200ldu_ctx_device_mem.argtypes = [vp, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    L.b200ldu_controls_default.argtypes = [C.POINTER(Controls)]
    L.b200ldu_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.b200ldu_ctx_destroy.argtypes = [vp]
    L.b200ldu_comm_unique_id.argtypes = [vp]
    L.b200ldu_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
    L.b200ldu_comm_info.argtypes = [vp, vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.b200ldu_ctx_set_stream.argtypes = [vp, vp]
    L.b200ldu_ctx_sync.argtypes = [vp]
    L.b200ldu_addr_create.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, C.POINTER(vp)]
    L.b200ldu_addr_destroy.argtypes = [vp]
    L.b200ldu_addr_info.argtypes = [vp, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong),
                                    C.POINTER(C.c_longlong), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.b200ldu_addr_face_info.argtypes = [vp, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong), C.POINTER(C.c_int),
                                         C.POINTER(C.c_int)]
    L.b200ldu_addr_face_templates.argtypes = [vp, C.POINTER(C.c_longlong), C.POINTER(C.c_int)]
    L.b200ldu_addr_perm.argtypes = [vp, vp]
    L.b200ldu_matrix_create.argtypes = [vp, C.POINTER(vp)]
    L.b200ldu_matrix_set.argtypes = [vp, vp, vp, vp, vp, vp]
    L.b200ldu_matrix_destroy.argtypes = [vp]
    for nm in ("b200ldu_amul", "b200ldu_tmul", "b200ldu_H", "b200ldu_faceH", "b200ldu_amul_banded",
               "b200ldu_to_banded", "b200ldu_from_banded"):
        getattr(L, nm).argtypes = [vp, vp, vp]
    L.b200ldu_sumA.argtypes = [vp, vp]
    L.b200ldu_H1.argtypes = [vp, vp]
    L.b200ldu_residual.argtypes = [vp, vp, vp, vp]
    L.b200ldu_precondition.argtypes = [vp, C.c_char_p, C.c_int, vp, vp]
    L.b200ldu_smooth.argtypes = [vp, C.c_char_p, C.c_double, vp, vp, C.c_int]
    L.b200ldu_solve.argtypes = [vp, C.c_char_p, C.c_char_p, C.POINTER(Controls), vp, vp, vp,
                                C.POINTER(Perf), vp, C.c_int]
    L.b200ldu_solve_host.argtypes = L.b200ldu_solve.argtypes
    L.b200ldu_bench_op.argtypes = [vp, C.c_char_p, vp, vp, vp]
    L.b200ldu_gamg_create.argtypes = [vp, vp, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(vp)]
    L.b200ldu_gamg_destroy.argtypes = [vp]
    L.b200ldu_gamg_nlevels.argtypes = [vp]
    L.b200ldu_gamg_level_size.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.b200ldu_gamg_restrict_addr.argtypes = [vp, C.c_int, vp]
    L.b200ldu_matrix_debug_trace.argtypes = [vp, C.c_int]
    L.b200ldu_matrix_debug_get.restype = C.c_longlong
    L.b200ldu_matrix_debug_get.argtypes = [vp, C.c_int, vp, C.c_longlong]
    L.b200ldu_gamg_debug_get.restype = C.c_longlong
    L.b200ldu_gamg_debug_get.argtypes = [vp, C.c_int, C.c_int, vp, C.c_longlong]
    L.b200ldu_gamg_debug_invert.argtypes = [C.c_int, vp, vp]
    L.b200ldu_fv_boundary_set.argtypes = [vp, C.c_int, vp]
    L.b200ldu_fv_surface_integrate.argtypes = [vp, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int]
    L.b200ldu_fv_gauss_grad.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp]
    L.b200ldu_fv_laplacian_fill.argtypes = [vp, vp, vp, vp, vp]
    L.b200ldu_fv_convection_fill.argtypes = [vp, vp, vp, vp, vp, vp]
    L.b200ldu_fv_interpolate_linear.argtypes = [vp, C.c_int, vp, vp, vp]
    L.b200ldu_fv_grad_linear.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.b200ldu_fv_flux_linear.argtypes = [vp, vp, vp, vp, vp]
    L.b200ldu_fv_add_boundary_diag.argtypes = [vp, vp, vp]
    L.b200ldu_fv_add_boundary_source.argtypes = [vp, vp, vp]
    L.b200ldu_fvm_add_boundary_diag.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
    L.b200ldu_fvm_add_boundary_source.argtypes = [vp, C.c_int, vp, vp, vp, vp]
    L.b200ldu_fvm_A.argtypes = [vp, C.c_int, vp, vp, vp]
    L.b200ldu_fvm_H.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp]
    L.b200ldu_fvm_flux.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp]
    L.b200ldu_fvm_residual.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.b200ldu_fvm_relax.argtypes = [vp, C.c_int, C.c_double, vp, vp, vp, vp]
    L.b200ldu_fvm_set_reference.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
    L.b200ldu_fv_patch_neighbour_field.argtypes = [vp, C.c_int, vp, vp]
    L.b200ldu_fv_sngrad.argtypes = [vp, C.c_int, vp, vp, vp]
    L.b200ldu_mules_limiter.argtypes = [vp, C.c_int, C.c_double] + [vp] * 12 + [C.c_double, C.c_double, vp, vp, C.c_int]
    L.b200ldu_mules_limiter_corr.argtypes = [vp, C.c_int, C.c_double] + [vp] * 9 + [C.c_double] * 3 + [vp, vp, C.c_int]
    L.b200ldu_ldu_row_sum.argtypes = [vp, C.c_int, vp, vp, vp]
    L.b200ldu_ldu_add_assign.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp]
    L.b200ldu_ldu_scale.argtypes = [vp, vp, C.c_double, vp, vp, vp, vp]
    L.b200ldu_fv_limiter.argtypes = [vp, C.c_char_p, C.c_double, vp, vp, vp, vp, vp]
    L.b200ldu_fv_limited_weights.argtypes = [vp, C.c_longlong, vp, vp, vp, vp]
    L.b200ldu_fv_limited_flux.argtypes = [vp, C.c_char_p, C.c_double, vp, vp, vp, vp, vp, C.c_int, C.c_int, vp]
    L.b200ldu_vof_interface_flux.argtypes = [vp] * 6 + [C.c_double, vp, vp, C.c_double, vp, vp, vp]
    L.b200ldu_field_binary.argtypes = [vp, C.c_int, C.c_longlong, C.c_int, vp, C.c_int, vp, vp]
    L.b200ldu_field_unary.argtypes = [vp, C.c_int, C.c_longlong, C.c_double, vp, vp]
    L.b200ldu_field_dot3.argtypes = [vp, C.c_longlong, vp, vp, vp]
    L.b200ldu_field_symm_magsqr.argtypes = [vp, C.c_longlong, vp, vp]
    L.b200ldu_field_gather.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
    L.b200ldu_fvm_set_values.argtypes = [vp, C.c_int] + [vp] * 9
    L.b200ldu_wallfn_nutk.argtypes = [vp, C.c_int, vp, vp, vp] + [C.c_double] * 5 + [vp]
    L.b200ldu_wallfn_epsilon.argtypes = [vp] + [vp] * 7 + [C.c_double] * 4 + [vp] * 3
    L.b200ldu_fvm_solve.argtypes = [vp, C.c_int, C.c_char_p, C.c_char_p, C.POINTER(Controls), vp, vp, vp, vp, vp, vp,
                                    C.POINTER(Perf)]
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise B200LduError(rc, lib().b200ldu_last_error().decode(errors="replace"))


def controls(**kw):
    c = Controls()
    lib().b200ldu_controls_default(C.byref(c))
    for k, v in kw.items():
        if not hasattr(c, k):
            raise KeyError(k)
        setattr(c, k, v)
    return c


def _np_i32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.int32)


def _np_f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


def _hp(a):
    return None if a is None else a.ctypes.data_as(vp)


def _dp(t):
    """device pointer of a torch cuda float64/int32 tensor (or None)"""
    if t is None:
        return None
    if not t.is_cuda or not t.is_contiguous():
        raise ValueError("device pointers must come from contiguous CUDA tensors")
    return vp(t.data_ptr())


class Context:
    """One per GPU (replaces argList's device selection and the Pstream communicator)."""

    def __init__(self, device=0, use_torch_stream=True):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("b200ldu needs a CUDA device; there is no CPU fallback")
        self.h = vp()
        check(lib().b200ldu_ctx_create(device, C.byref(self.h)))
        self.device = torch.device("cuda", device)
        if use_torch_stream:
            check(lib().b200ldu_ctx_set_stream(self.h, vp(torch.cuda.current_stream(self.device).cuda_stream)))
        self.rank, self.nRanks = 0, 1

    def comm_init_from_torch(self):
        """Create the NCCL communicator; the unique id travels over torch.distributed."""
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(), dist.get_world_size()
        buf = (C.c_char * 128)()
        if rank == 0:
            check(lib().b200ldu_comm_unique_id(C.cast(buf, vp)))
        t = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
        if dist.get_backend() == "nccl":
            t = t.to(self.device)
        dist.broadcast(t, 0)
        raw = bytes(t.cpu().numpy().tobytes())
        idbuf = C.create_string_buffer(raw, 128)
        check(lib().b200ldu_comm_init(self.h, C.cast(idbuf, vp), rank, world))
        self.rank, self.nRanks = rank, world

    def sync(self):
        check(lib().b200ldu_ctx_sync(self.h))

    @property
    def launches(self):
        return lib().b200ldu_launch_count(self.h)

    def close(self):
        if self.h:
            lib().b200ldu_ctx_destroy(self.h)
            self.h = vp()


class LduAddressing:
    """lduAddressing (+ coupled patches) -> banded device layout."""

    def __init__(self, ctx, nCells, lower, upper, patchStart=None, faceCells=None, neighbRank=None,
                 cellCentres=None):
        self.ctx = ctx
        self.nCells = int(nCells)
        l, u = _np_i32(lower), _np_i32(upper)
        self.nFaces = len(l)
        ps, fc, nr = _np_i32(patchStart), _np_i32(faceCells), _np_i32(neighbRank)
        nP = 0 if ps is None else len(ps) - 1
        self.nPatchFaces = 0 if ps is None else int(ps[-1])
        cc = _np_f64(cellCentres)
        self.h = vp()
        check(lib().b200ldu_addr_create(ctx.h, self.nCells, self.nFaces, _hp(l), _hp(u), nP, _hp(ps), _hp(fc),
                                        _hp(nr), _hp(cc), C.byref(self.h)))

    def info(self):
        a, b, c = C.c_longlong(), C.c_longlong(), C.c_longlong()
        d, e = C.c_int(), C.c_int()
        check(lib().b200ldu_addr_info(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d), C.byref(e)))
        fo, fl, fb, fu = C.c_longlong(), C.c_longlong(), C.c_int(), C.c_int()
        check(lib().b200ldu_addr_face_info(self.h, C.byref(fo), C.byref(fl), C.byref(fb), C.byref(fu)))
        tw, tc = C.c_longlong(), C.c_int()
        check(lib().b200ldu_addr_face_templates(self.h, C.byref(tw), C.byref(tc)))
        return dict(nPadRows=a.value, nEntries=b.value, nHalo=c.value, bandRows=d.value, nBands=e.value,
                    fsOwnerSlots=fo.value, fsListItems=fl.value, fsBufDoubles=fb.value, faceStream=bool(fu.value),
                    fsTemplateWords=tw.value, fsTemplates=tc.value)

    def perm(self):
        p = np.zeros(self.nCells, dtype=np.int32)
        check(lib().b200ldu_addr_perm(self.h, _hp(p)))
        return p

    @property
    def vec_len(self):
        return lib().b200ldu_vec_len(self.h)

    def close(self):
        if self.h:
            lib().b200ldu_addr_destroy(self.h)
            self.h = vp()


class LduMatrix:
    """lduMatrix: coefficients in banded form + the operations the solvers consume."""

    def __init__(self, addr):
        self.addr = addr
        self.h = vp()
        check(lib().b200ldu_matrix_create(addr.h, C.byref(self.h)))
        self._keep = None

    def set(self, diag, upper, lower=None, bouCoeffs=None, intCoeffs=None):
        self._keep = (diag, upper, lower, bouCoeffs, intCoeffs)  # faceH reads upper/lower later
        check(lib().b200ldu_matrix_set(self.h, _dp(diag), _dp(upper), _dp(lower), _dp(bouCoeffs), _dp(intCoeffs)))
        return self

    def _new(self, like, n=None):
        import torch
        return torch.empty(like.shape[0] if n is None else n, dtype=torch.float64, device=like.device)

    def Amul(self, psi):
        out = self._new(psi)
        check(lib().b200ldu_amul(self.h, _dp(psi), _dp(out)))
        return out

    def Tmul(self, psi):
        out = self._new(psi)
        check(lib().b200ldu_tmul(self.h, _dp(psi), _dp(out)))
        return out

    def sumA(self, like):
        out = self._new(like)
        check(lib().b200ldu_sumA(self.h, _dp(out)))
        return out

    def residual(self, psi, source):
        out = self._new(psi)
        check(lib().b200ldu_residual(self.h, _dp(psi), _dp(source), _dp(out)))
        return out

    def H(self, psi):
        out = self._new(psi)
        check(lib().b200ldu_H(self.h, _dp(psi), _dp(out)))
        return out

    def H1(self, like):
        out = self._new(like)
        check(lib().b200ldu_H1(self.h, _dp(out)))
        return out

    def faceH(self, psi):
        out = self._new(psi, self.addr.nFaces)
        check(lib().b200ldu_faceH(self.h, _dp(psi), _dp(out)))
        return out

    def precondition(self, name, rA, transpose=False):
        out = self._new(rA)
        check(lib().b200ldu_precondition(self.h, name.encode(), int(transpose), _dp(rA), _dp(out)))
        return out

    def smooth(self, name, psi, source, nSweeps, omega=0.9):
        p = psi.clone()
        check(lib().b200ldu_smooth(self.h, name.encode(), omega, _dp(p), _dp(source), nSweeps))
        return p

    def solve(self, solver, pre, psi, source, gamg=None, histCap=0, **ctl):
        """lduMatrix::solver::New(...)->solve(psi, source): psi updated in place.
        Returns (Perf, history ndarray)."""
        c = controls(**ctl)
        perf = Perf()
        hist = np.full(max(histCap, 1), np.nan)
        check(lib().b200ldu_solve(self.h, solver.encode(), (pre or "").encode(), C.byref(c),
                                  gamg.h if gamg is not None else None, _dp(psi), _dp(source),
                                  C.byref(perf), _hp(hist) if histCap else None, histCap))
        return perf, hist[~np.isnan(hist)] if histCap else hist[:0]

    # b200ldu_matrix_debug_get's codes, and the step kinds of a trace record (B200LDU_STEP_*), in order
    TRACE_WHAT = ("records", "partials", "scalars")
    STEP_KINDS = ("other", "init", "norm", "beta", "alpha", "end", "pcgA", "pcgB", "pcgClose", "rho", "rA0AyA",
                  "sMag", "omega")
    SCALARS = ("wArA", "wApA", "alpha", "beta", "omega", "rA0rA", "tAtA", "tAsA", "normFactor", "bodies", "psiBodies",
               "steps")

    def debug_trace(self, cap):
        """Record the global sums of this handle's later solves, up to cap scalar steps per solve (0: stop)."""
        check(lib().b200ldu_matrix_debug_trace(self.h, int(cap)))

    def debug_get(self, name):
        """HOST copy of the last solve's trace (b200ldu_matrix_debug_get): "records" float64[nRec, 16],
        "partials" float64[nRec, P], or "scalars" as a dict of the final SolverScalars fields"""
        what = self.TRACE_WHAT.index(name)
        n = lib().b200ldu_matrix_debug_get(self.h, what, None, 0)
        check(int(min(0, n)))
        out = np.zeros(max(n, 1))
        check(int(min(0, lib().b200ldu_matrix_debug_get(self.h, what, _hp(out), n))))
        out = out[:n]
        if name == "scalars":
            return dict(zip(self.SCALARS, out.tolist()))
        if name == "records":
            return out.reshape(-1, 16)
        nRec = len(self.debug_get("records"))
        return out.reshape(nRec, -1) if nRec else out.reshape(0, 0)

    def solve_host(self, solver, pre, psi_h, source_h, gamg=None, **ctl):
        """End-to-end entry: HOST numpy psi/source, H2D + solve + D2H inside the call."""
        c = controls(**ctl)
        perf = Perf()
        assert psi_h.dtype == np.float64 and source_h.dtype == np.float64
        check(lib().b200ldu_solve_host(self.h, solver.encode(), (pre or "").encode(), C.byref(c),
                                       gamg.h if gamg is not None else None, _hp(psi_h), _hp(source_h),
                                       C.byref(perf), None, 0))
        return perf

    def close(self):
        if self.h:
            lib().b200ldu_matrix_destroy(self.h)
            self.h = vp()


class FvMatrix:
    """fvMatrix<Type> around an LduMatrix (FV/fvMatrices/fvMatrix/fvMatrix.H; SURVEY.md section 8 row a17), with
    the reference's member names.  Type = scalar (nComp 1) or vector (nComp 3); fields are device tensors with
    the components interleaved.  The non-coupled boundary faces are the flat list given to
    b200ldu_fv_boundary_set; internalCoeffs / boundaryCoeffs hold nBFaces*nComp values.  Coupled patches take their
    coefficients from the LduMatrix (set(..., bouCoeffs, intCoeffs)) and their patchNeighbourField from `pnf`."""

    def __init__(self, matrix, nComp, diag, source, psi, V, internalCoeffs=None, boundaryCoeffs=None):
        self.m, self.nc = matrix, int(nComp)
        self.diag, self.source, self.psi, self.V = diag, source, psi, V
        self.ic, self.bc = internalCoeffs, boundaryCoeffs

    def _new(self, n):
        import torch
        return torch.empty(n, dtype=torch.float64, device=self.psi.device)

    def addBoundaryDiag(self, diag, cmpt):
        check(lib().b200ldu_fvm_add_boundary_diag(self.m.h, self.nc, cmpt, _dp(self.ic), _dp(diag), _dp(diag)))

    def addCmptAvBoundaryDiag(self, diag):
        check(lib().b200ldu_fvm_add_boundary_diag(self.m.h, self.nc, -1, _dp(self.ic), _dp(diag), _dp(diag)))

    def addBoundarySource(self, source, pnf=None):
        check(lib().b200ldu_fvm_add_boundary_source(self.m.h, self.nc, _dp(self.bc), _dp(pnf), _dp(source), _dp(source)))

    def A(self):
        out = self._new(self.m.addr.nCells)
        check(lib().b200ldu_fvm_A(self.m.h, self.nc, _dp(self.ic), _dp(self.V), _dp(out)))
        return out

    def H(self, pnf=None):
        out = self._new(self.m.addr.nCells * self.nc)
        check(lib().b200ldu_fvm_H(self.m.h, self.nc, _dp(self.psi), _dp(self.source), _dp(self.bc), _dp(pnf),
                                  _dp(self.V), _dp(out)))
        return out

    def flux(self, nBFaces, nCoupledFaces=0, pnf=None):
        """(internal faces, non-coupled boundary faces, coupled faces), each with nComp values per face"""
        f = self._new(max(self.m.addr.nFaces * self.nc, 1))
        b = self._new(max(nBFaces * self.nc, 1))
        c = self._new(max(nCoupledFaces * self.nc, 1))
        check(lib().b200ldu_fvm_flux(self.m.h, self.nc, _dp(self.psi), _dp(self.ic), _dp(self.bc), _dp(pnf), _dp(f),
                                     _dp(b), _dp(c)))
        return f[: self.m.addr.nFaces * self.nc], b[: nBFaces * self.nc], c[: nCoupledFaces * self.nc]

    def residual(self, pnf=None):
        out = self._new(self.m.addr.nCells)
        check(lib().b200ldu_fvm_residual(self.m.h, _dp(self.psi), _dp(self.source), _dp(self.ic), _dp(self.bc),
                                         _dp(pnf), _dp(out)))
        return out

    def relax(self, alpha):
        """in place on diag and source; the LduMatrix has to be set() again before it is used"""
        check(lib().b200ldu_fvm_relax(self.m.h, self.nc, float(alpha), _dp(self.psi), _dp(self.ic), _dp(self.diag),
                                      _dp(self.source)))

    def setReference(self, celli, value):
        v = np.ascontiguousarray(np.atleast_1d(np.asarray(value, np.float64)))
        check(lib().b200ldu_fvm_set_reference(self.m.h, int(celli), self.nc, _hp(v), _dp(self.diag), _dp(self.source)))

    def setValues(self, cells, values, upper, lower):
        """fvMatrix::setValues (scalar, single domain), in place on psi, source, upper, lower, internalCoeffs and
        boundaryCoeffs; `lower` is required (a copy of upper for a symmetric matrix: the result is asymmetric, see
        b200ldu.h).  cells: int32 device tensor, a cell listed twice with equal values.  The LduMatrix has to be set()
        again before it is used."""
        check(lib().b200ldu_fvm_set_values(self.m.h, cells.numel(), _dp(cells), _dp(values), _dp(self.psi), _dp(self.diag),
                                           _dp(upper), _dp(lower), _dp(self.source), _dp(self.ic), _dp(self.bc)))

    def solve(self, solver, pre, gamg=None, pnf=None, **ctl):
        """solveSegregated: psi updated in place; returns the list of Perf, one per component"""
        c = controls(**ctl)
        perfs = (Perf * self.nc)()
        check(lib().b200ldu_fvm_solve(self.m.h, self.nc, solver.encode(), (pre or "").encode(), C.byref(c),
                                      gamg.h if gamg is not None else None, _dp(self.psi), _dp(self.source),
                                      _dp(self.ic), _dp(self.bc), _dp(pnf), perfs))
        return list(perfs)


class GamgAgglomeration:
    def __init__(self, addr, faceWeights, nCellsInCoarsestLevel=10, mergeLevels=1, forward=1):
        self.addr = addr
        self.h = vp()
        self._fw = C.c_int(int(forward))
        w = _np_f64(faceWeights)
        check(lib().b200ldu_gamg_create(addr.h, _hp(w), nCellsInCoarsestLevel, mergeLevels, C.byref(self._fw),
                                        C.byref(self.h)))
        self.nLevels = lib().b200ldu_gamg_nlevels(self.h)

    @property
    def forward(self):
        return self._fw.value

    def level_size(self, lev):
        a, b = C.c_int(), C.c_int()
        check(lib().b200ldu_gamg_level_size(self.h, lev, C.byref(a), C.byref(b)))
        return a.value, b.value

    def restrict_addr(self, lev):
        n = self.addr.nCells if lev == 0 else self.level_size(lev - 1)[0]
        out = np.zeros(n, dtype=np.int32)
        check(lib().b200ldu_gamg_restrict_addr(self.h, lev, _hp(out)))
        return out

    # b200ldu_gamg_debug_get's codes, in order, with the element type of each
    DEBUG = [("owner", np.int32), ("neighbour", np.int32), ("faceRestrict", np.int32), ("faceFlip", np.int32),
             ("diag", np.float64), ("upper", np.float64), ("lower", np.float64), ("bou", np.float64),
             ("int", np.float64), ("perm", np.int32), ("inv", np.float64), ("invDims", np.int32)]

    def debug_get(self, lev, name):
        """HOST copy of one array of coarse level lev (b200ldu_gamg_debug_get)"""
        what = [k for k, _ in self.DEBUG].index(name)
        n = lib().b200ldu_gamg_debug_get(self.h, lev, what, None, 0)
        if n < 0:
            check(int(n))
        out = np.zeros(max(n, 1), dtype=self.DEBUG[what][1])
        check(int(min(0, lib().b200ldu_gamg_debug_get(self.h, lev, what, _hp(out), n))))
        return out[:n]

    def level_addressing(self, lev):
        """dict(owner, neighbour, faceRestrict, faceFlip) of coarse level lev; also on a host-only hierarchy"""
        return {k: self.debug_get(lev, k) for k in ("owner", "neighbour", "faceRestrict", "faceFlip")}

    def level_state(self, lev):
        """the addressing, the last solve's coarse coefficients (lower None when that matrix was symmetric), the
        interface coefficients and the banded permutation of coarse level lev"""
        out = self.level_addressing(lev)
        for k in ("diag", "upper", "lower", "bou", "int", "perm"):
            out[k] = self.debug_get(lev, k)
        if out["lower"].size == 0 and out["upper"].size:
            out["lower"] = None
        return out

    def coarsest_inverse(self):
        """(rows, N, offset): this rank's rows of the inverse of the coarsest matrix as the last solve uploaded
        them -- banded rows x global banded columns -- the global size and this rank's first row"""
        lev = self.nLevels - 1
        N, off, n = (int(v) for v in self.debug_get(lev, "invDims"))
        return self.debug_get(lev, "inv").reshape(n, N), N, off

    def close(self):
        if self.h:
            lib().b200ldu_gamg_destroy(self.h)
            self.h = vp()


class FieldOps:
    """The gpuField operator set between the kernels (b200ldu_field_*): one rounded operation per call, composed by
    the caller in the reference's order.  Fields are flat device tensors; nc* = components per element."""
    ADD, SUB, MUL, DIV, MIN, MAX = range(6)

    def __init__(self, ctx):
        self.ctx = ctx

    def _new(self, like, n):
        import torch
        return torch.empty(n, dtype=torch.float64, device=like.device)

    def binary(self, op, a, b, nca=1, ncb=1):
        n = a.numel() // nca
        assert b.numel() // ncb == n
        out = self._new(a, n * max(nca, ncb))
        check(lib().b200ldu_field_binary(self.ctx.h, op, n, nca, _dp(a), ncb, _dp(b), _dp(out)))
        return out

    def add(self, a, b, nca=1, ncb=1):
        return self.binary(self.ADD, a, b, nca, ncb)

    def sub(self, a, b, nca=1, ncb=1):
        return self.binary(self.SUB, a, b, nca, ncb)

    def mul(self, a, b, nca=1, ncb=1):
        return self.binary(self.MUL, a, b, nca, ncb)

    def div(self, a, b, nca=1, ncb=1):
        return self.binary(self.DIV, a, b, nca, ncb)

    def unary(self, op, a, s=0.0):
        out = self._new(a, a.numel())
        check(lib().b200ldu_field_unary(self.ctx.h, op, a.numel(), float(s), _dp(a), _dp(out)))
        return out

    def neg(self, a):
        return self.unary(0, a)

    def mag(self, a):
        return self.unary(1, a)

    def smul(self, s, a):            # s*a
        return self.unary(2, a, s)

    def rdiv(self, s, a):            # s/a
        return self.unary(3, a, s)

    def sadd(self, a, s):            # a + s
        return self.unary(4, a, s)

    def rsub(self, s, a):            # s - a
        return self.unary(5, a, s)

    def smin(self, a, s):            # min(a, s)
        return self.unary(6, a, s)

    def sdiv(self, a, s):            # a/s
        return self.unary(9, a, s)

    def smax(self, a, s):            # max(a, s)
        return self.unary(7, a, s)

    def pos(self, a):                # pos(a): 1 where a >= 0, else 0
        return self.unary(11, a)

    def bmax(self, a, b):            # max(a, b) per element
        return self.binary(self.MAX, a, b)

    def symm_magsqr(self, T):        # magSqr(symm(T)), T [n*9]
        out = self._new(T, T.numel() // 9)
        check(lib().b200ldu_field_symm_magsqr(self.ctx.h, T.numel() // 9, _dp(T), _dp(out)))
        return out

    def dot3(self, a, b):
        out = self._new(a, a.numel() // 3)
        check(lib().b200ldu_field_dot3(self.ctx.h, a.numel() // 3, _dp(a), _dp(b), _dp(out)))
        return out

    def gather(self, cells, f, nc=1):
        out = self._new(f, cells.numel() * nc)
        check(lib().b200ldu_field_gather(self.ctx.h, cells.numel(), nc, _dp(cells), _dp(f), _dp(out)))
        return out


def _newlike(t, n):
    import torch
    return torch.empty(n, dtype=torch.float64, device=t.device)


def wallfn_nutk(addr, faces, y, k, nuw, yPlusLam, Cmu25, nutB, kappa=0.41, E=9.8):
    """nutkWallFunction::calcNut into nutB at the boundary faces `faces` (int32 device tensor), in place"""
    check(lib().b200ldu_wallfn_nutk(addr.h, faces.numel(), _dp(faces), _dp(y), _dp(k), float(nuw), float(yPlusLam), float(Cmu25),
                                    float(kappa), float(E), _dp(nutB)))


def wallfn_epsilon(addr, cornerWeights, y, k, U, Ub, bDelta, nutB, nu, Cmu25, Cmu75, G, epsilon, epsB, kappa=0.41):
    """epsilonWallFunction::updateCoeffs of all epsilon-wall patches: G, epsilon and epsB in place (b200ldu.h)"""
    check(lib().b200ldu_wallfn_epsilon(addr.h, _dp(cornerWeights), _dp(y), _dp(k), _dp(U), _dp(Ub), _dp(bDelta), _dp(nutB),
                                       float(nu), float(Cmu25), float(Cmu75), float(kappa), _dp(G), _dp(epsilon), _dp(epsB)))


def fv_convection_fill(addr, weights, phi):
    """gaussConvectionScheme::fvmDiv coefficients: (lower, upper, diag)"""
    lo, up, dg = _newlike(phi, addr.nFaces), _newlike(phi, addr.nFaces), _newlike(phi, addr.nCells)
    check(lib().b200ldu_fv_convection_fill(addr.h, _dp(weights), _dp(phi), _dp(lo), _dp(up), _dp(dg)))
    return lo, up, dg


def fv_laplacian_fill(addr, deltaCoeffs, gammaMagSf):
    """gaussLaplacianScheme::fvmLaplacianUncorrected coefficients: (upper, diag)"""
    up, dg = _newlike(gammaMagSf, addr.nFaces), _newlike(gammaMagSf, addr.nCells)
    check(lib().b200ldu_fv_laplacian_fill(addr.h, _dp(deltaCoeffs), _dp(gammaMagSf), _dp(up), _dp(dg)))
    return up, dg


def fv_interpolate_linear(addr, nComp, w, vf):
    sf = _newlike(vf, addr.nFaces * nComp)
    check(lib().b200ldu_fv_interpolate_linear(addr.h, nComp, _dp(w), _dp(vf), _dp(sf)))
    return sf


def fv_flux_linear(addr, Sf, w, U):
    """interpolate(U) & Sf per internal face"""
    phi = _newlike(U, addr.nFaces)
    check(lib().b200ldu_fv_flux_linear(addr.h, _dp(Sf), _dp(w), _dp(U), _dp(phi)))
    return phi


def fv_grad_linear(addr, nComp, Sf, w, vf, bSf, bvf, V):
    """gaussGrad(linear): gradf(interpolate(vf)) without the face field"""
    g = _newlike(vf, addr.nCells * 3 * nComp)
    check(lib().b200ldu_fv_grad_linear(addr.h, nComp, _dp(Sf), _dp(w), _dp(vf), _dp(bSf), _dp(bvf), _dp(V), _dp(g)))
    return g


def fv_surface_integrate(addr, nComp, ssf, bssf, V, divideByV=True, neiSign=-1):
    out = _newlike(ssf, addr.nCells * nComp)
    check(lib().b200ldu_fv_surface_integrate(addr.h, nComp, _dp(ssf), _dp(bssf), _dp(V), _dp(out), int(divideByV), neiSign))
    return out


def fv_patch_neighbour_field(addr, nComp, field):
    """coupledFvPatchField::patchNeighbourField of every coupled patch face (processor: exchanged, cyclic: partner)"""
    pnf = _newlike(field, max(addr.nPatchFaces * nComp, 1))
    check(lib().b200ldu_fv_patch_neighbour_field(addr.h, nComp, _dp(field), _dp(pnf)))
    return pnf[: addr.nPatchFaces * nComp]


def fv_sngrad(addr, nComp, deltaCoeffs, vf):
    """snGradScheme::snGrad on the internal faces"""
    out = _newlike(vf, addr.nFaces * nComp)
    check(lib().b200ldu_fv_sngrad(addr.h, nComp, _dp(deltaCoeffs), _dp(vf), _dp(out)))
    return out


class LduCoeffs:
    """diag / upper / lower device arrays with presence flags: the optional arrays of the reference's lduMatrix, for
    the algebra of lduMatrixOperations.C (sumDiag ..., operator+= -= *=)"""

    def __init__(self, addr, diag=None, upper=None, lower=None):
        import torch
        self.addr = addr
        dev = addr.ctx.device
        z = lambda n: torch.zeros(max(n, 1), dtype=torch.float64, device=dev)
        self.has = (C.c_int * 3)(diag is not None, upper is not None, lower is not None)
        self.diag = diag.clone() if diag is not None else z(addr.nCells)
        self.upper = upper.clone() if upper is not None else z(addr.nFaces)
        self.lower = lower.clone() if lower is not None else z(addr.nFaces)

    def _combine(self, other, sub):
        check(lib().b200ldu_ldu_add_assign(self.addr.h, sub, _dp(self.diag), _dp(self.upper), _dp(self.lower), self.has,
                                           _dp(other.diag), _dp(other.upper), _dp(other.lower), other.has))
        return self

    def __iadd__(self, other):
        return self._combine(other, 0)

    def __isub__(self, other):
        return self._combine(other, 1)

    def scale(self, s):
        """*= a cell field (tensor) or a scalar"""
        sf = None if isinstance(s, (int, float)) else s
        check(lib().b200ldu_ldu_scale(self.addr.h, _dp(sf), float(s) if sf is None else 0.0, _dp(self.diag), _dp(self.upper),
                                      _dp(self.lower), self.has))
        return self

    def row_sum(self, mode, inout):
        """0 sumDiag, 1 negSumDiag, 2 sumMagOffDiag; in place on `inout`"""
        check(lib().b200ldu_ldu_row_sum(self.addr.h, mode, _dp(self.upper) if self.has[1] else _dp(self.lower),
                                        _dp(self.lower) if self.has[2] else None, _dp(inout)))
        return inout

    def arrays(self):
        return (self.diag[: self.addr.nCells] if self.has[0] else None, self.upper[: self.addr.nFaces] if self.has[1] else None,
                self.lower[: self.addr.nFaces] if self.has[2] else None)


def fv_limiter(addr, scheme, faceFlux, vf, gradc, centres, k=1.0):
    """limiter field of a limited scheme on the internal faces (LimitedScheme::calcLimiter)"""
    out = _newlike(faceFlux, addr.nFaces)
    check(lib().b200ldu_fv_limiter(addr.h, scheme.encode(), float(k), _dp(faceFlux), _dp(vf), _dp(gradc), _dp(centres), _dp(out)))
    return out


def fv_limited_weights(ctx, faceFlux, limiter=None, cdWeights=None):
    """interpolation weights of a limited scheme; limiter None: upwind, pos(faceFlux)"""
    out = _newlike(faceFlux, faceFlux.numel())
    check(lib().b200ldu_fv_limited_weights(ctx.h, faceFlux.numel(), _dp(limiter), _dp(cdWeights), _dp(faceFlux), _dp(out)))
    return out


def fv_limited_flux(addr, scheme, faceFlux, vf, gradc, centres, cdWeights, k=1.0, fluxSign=1, outSign=1):
    """outSign*fvc::flux(fluxSign*faceFlux, vf, scheme) on the internal faces in one pass: limiter, weights, face value and the
    product with the flux, bit for bit the composition of fv_limiter, fv_limited_weights, fv_interpolate_linear and a multiply"""
    out = _newlike(faceFlux, addr.nFaces)
    check(lib().b200ldu_fv_limited_flux(addr.h, scheme.encode(), float(k), _dp(faceFlux), _dp(vf), _dp(gradc), _dp(centres),
                                        _dp(cdWeights), int(fluxSign), int(outSign), _dp(out)))
    return out


def vof_interface_flux(addr, w, gradAlpha, Sf, bSf, bSnGrad, deltaN, phi=None, magSf=None, cAlpha=0.0):
    """interfaceProperties::calculateK up to nHatf, and the compression flux: (nHatf on the internal faces, nHatf on the boundary
    faces of fv_boundary_set, phir = cAlpha*|phi/magSf|*nHatf on the internal faces or None without phi)"""
    nB = 0 if bSnGrad is None else bSnGrad.numel()
    nHatf, nHatfB = _newlike(w, addr.nFaces), _newlike(w, max(nB, 1))
    phir = None if phi is None else _newlike(w, addr.nFaces)
    check(lib().b200ldu_vof_interface_flux(addr.h, _dp(w), _dp(gradAlpha), _dp(Sf), _dp(bSf), _dp(bSnGrad), float(deltaN), _dp(phi),
                                           _dp(magSf), float(cAlpha), _dp(nHatf), _dp(nHatfB), _dp(phir)))
    return nHatf, nHatfB[:nB], phir


def mules_limiter(addr, V, rDeltaT, psi, psi0, psiB, phiBD, phiBDB, phiCorr, phiCorrB, psiMax, psiMin, nLimiterIter=3,
                  rho=None, rho0=None, Sp=None, Su=None, nCoupled=0):
    """MULES::limiter: (lambda on the internal faces, lambda on the boundary faces of fv_boundary_set), starting from 1.  nCoupled:
    the trailing boundary faces that are coupled patch faces (psiB = patchNeighbourField there); collective over the ranks"""
    import torch
    lam = torch.ones(addr.nFaces, dtype=torch.float64, device=psi.device)
    lamB = torch.ones(max(phiCorrB.numel(), 1), dtype=torch.float64, device=psi.device)
    check(lib().b200ldu_mules_limiter(addr.h, int(nLimiterIter), float(rDeltaT), _dp(rho), _dp(rho0), _dp(psi), _dp(psi0), _dp(psiB),
                                      _dp(phiBD), _dp(phiBDB), _dp(phiCorr), _dp(phiCorrB), _dp(Sp), _dp(Su), _dp(V), float(psiMax),
                                      float(psiMin), _dp(lam), _dp(lamB), int(nCoupled)))
    return lam, lamB[: phiCorrB.numel()]


def mules_limiter_corr(addr, V, rDeltaT, psi, psiB, phiB, phiCorr, phiCorrB, psiMax, psiMin, nLimiterIter=3, rho=None, Sp=None, Su=None,
                       extremaCoeff=0.0, nCoupled=0):
    """MULES::limiterCorr: the limiters of a flux correction, (internal faces, boundary faces of fv_boundary_set), starting from 1"""
    import torch
    lam = torch.ones(addr.nFaces, dtype=torch.float64, device=psi.device)
    lamB = torch.ones(max(phiCorrB.numel(), 1), dtype=torch.float64, device=psi.device)
    check(lib().b200ldu_mules_limiter_corr(addr.h, int(nLimiterIter), float(rDeltaT), _dp(rho), _dp(psi), _dp(psiB), _dp(phiB), _dp(phiCorr),
                                           _dp(phiCorrB), _dp(Sp), _dp(Su), _dp(V), float(psiMax), float(psiMin), float(extremaCoeff),
                                           _dp(lam), _dp(lamB), int(nCoupled)))
    return lam, lamB[: phiCorrB.numel()]


def fv_boundary_set(addr, bFaceCells):
    """the non-coupled boundary faces (all patches, patch order) of the FV face sums and the fvMatrix glue"""
    bfc = _np_i32(bFaceCells)
    check(lib().b200ldu_fv_boundary_set(addr.h, len(bfc), _hp(bfc)))


def mesh_to_device(ctx, mesh, with_centres=True):
    """LduAddressing for a rapidcfd-dev_b200.mesh.HexMesh (processor patches included)."""
    ps, fc = mesh.patch_start_facecells()
    nr = np.array([p.neighbRank for p in mesh.coupled_patches()], dtype=np.int32)
    if len(nr) == 0:
        ps = fc = nr = None
    return LduAddressing(ctx, mesh.nCells, mesh.lower, mesh.upper, ps, fc, nr,
                         mesh.cell_centres() if with_centres else None)


def polymesh_to_device(ctx, pm, cellCentres=None):
    """LduAddressing for a foamfile.PolyMesh read from constant/polyMesh (processor and cyclic
    patches included).  cellCentres: optional [nCells,3] (pm.fv_geometry()["C"]) for the renumbering."""
    lo, up = pm.ldu()
    ps, fc, nr = pm.coupled_interface_arrays()
    return LduAddressing(ctx, pm.nCells, lo, up, ps, fc, nr, cellCentres)

