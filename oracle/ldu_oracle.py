"""ctypes binding of the CPU oracle (oracle/ldu_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package (rapidcfd-dev_b200/) never
imports this module.  The reference has no tests of its own; what is pinned to its source code
(oracle/ref_ldu.py, tests/test_reference_functors.py) and what is not is listed in oracle/ldu_oracle.h.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "_build", "libldu_oracle.so")

c_dp = C.POINTER(C.c_double)
c_ip = C.POINTER(C.c_int)


def build(force=False):
    """Compile the oracle with the committed Makefile (gcc, -ffp-contract=off)."""
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h"))]
    if not force and os.path.exists(_LIB):
        if all(os.path.getmtime(s) <= os.path.getmtime(_LIB) for s in srcs):
            return _LIB
    subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB


class Controls(C.Structure):
    _fields_ = [
        ("tolerance", C.c_double), ("relTol", C.c_double),
        ("maxIter", C.c_int), ("minIter", C.c_int), ("nSweeps", C.c_int),
        ("omega", C.c_double), ("bicgstabRefQuirk", C.c_int),
        ("nCellsInCoarsestLevel", C.c_int), ("mergeLevels", C.c_int),
        ("nPreSweeps", C.c_int), ("preSweepsLevelMultiplier", C.c_int), ("maxPreSweeps", C.c_int),
        ("nPostSweeps", C.c_int), ("postSweepsLevelMultiplier", C.c_int), ("maxPostSweeps", C.c_int),
        ("nFinestSweeps", C.c_int), ("interpolateCorrection", C.c_int),
        ("scaleCorrection", C.c_int), ("directSolveCoarsest", C.c_int),
    ]


class Perf(C.Structure):
    _fields_ = [
        ("initialResidual", C.c_double), ("finalResidual", C.c_double), ("normFactor", C.c_double),
        ("nIterations", C.c_int), ("converged", C.c_int), ("singular", C.c_int),
        ("solverName", C.c_char * 64),
    ]


HALO_CB = C.CFUNCTYPE(None, C.c_void_p, c_dp, c_dp, C.c_int, C.c_int, c_ip)
SUM_CB = C.CFUNCTYPE(None, C.c_void_p, c_dp, C.c_int)
GATHER_CB = C.CFUNCTYPE(None, C.c_void_p, c_dp, C.c_int, c_dp)
REDUCE_CB = C.CFUNCTYPE(C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_int, c_dp, c_dp, C.c_int, C.c_double)

# call sites of the reduction hook, in the order of ORC_SITE_* (ldu_oracle.h), and its term kinds (ORC_RED_*)
SITES = ("sumPsi", "normFactor", "sumMag0", "wArA", "wApA", "sumMag", "wArT", "wApT", "rA0rA", "rA0AyA", "sumMagS",
         "tAtA", "tAsA")
RED_OPS = ("sum", "prod", "mag")


class Comm(C.Structure):
    _fields_ = [("ctx", C.c_void_p), ("halo", HALO_CB), ("sum", SUM_CB), ("nCellsGlobal", C.c_longlong),
                ("gather", GATHER_CB), ("rank", C.c_int), ("nRanks", C.c_int)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        L.orc_addr_create.restype = C.c_void_p
        L.orc_addr_create.argtypes = [C.c_int, C.c_int, c_ip, c_ip, C.c_int, c_ip, c_ip]
        L.orc_addr_free.argtypes = [C.c_void_p]
        for nm in ("orc_addr_owner_start", "orc_addr_losort", "orc_addr_losort_start", "orc_addr_lower",
                   "orc_addr_upper"):
            getattr(L, nm).restype = c_ip
            getattr(L, nm).argtypes = [C.c_void_p]
        L.orc_matrix_create.restype = C.c_void_p
        L.orc_matrix_create.argtypes = [C.c_void_p, c_dp, c_dp, c_dp, c_dp, c_dp]
        L.orc_matrix_free.argtypes = [C.c_void_p]
        L.orc_amul.argtypes = [C.c_void_p, c_dp, c_dp, C.c_void_p]
        L.orc_tmul.argtypes = [C.c_void_p, c_dp, c_dp, C.c_void_p]
        L.orc_sumA.argtypes = [C.c_void_p, c_dp]
        L.orc_residual.argtypes = [C.c_void_p, c_dp, c_dp, c_dp, C.c_void_p]
        L.orc_H.argtypes = [C.c_void_p, c_dp, c_dp]
        L.orc_H1.argtypes = [C.c_void_p, c_dp]
        L.orc_faceH.argtypes = [C.c_void_p, c_dp, c_dp]
        for nm in ("orc_sumDiag", "orc_negSumDiag", "orc_sumMagOffDiag"):
            getattr(L, nm).argtypes = [C.c_void_p, c_dp, c_dp, c_dp]
        L.orc_normFactor.restype = C.c_double
        L.orc_normFactor.argtypes = [C.c_void_p, c_dp, c_dp, c_dp, c_dp, C.c_void_p]
        L.orc_precondition.argtypes = [C.c_void_p, C.c_int, C.c_int, c_dp, c_dp, c_dp]
        L.orc_jacobi_smooth.argtypes = [C.c_void_p, C.c_double, c_dp, c_dp, C.c_int, C.c_void_p]
        L.orc_controls_default.argtypes = [C.POINTER(Controls)]
        L.orc_solve.restype = C.c_int
        L.orc_solve.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.POINTER(Controls), c_dp, c_dp,
                                C.c_void_p, C.POINTER(Perf), c_dp, C.c_int]
        L.orc_gamg_create.restype = C.c_void_p
        L.orc_gamg_create.argtypes = [C.c_void_p, c_dp, C.c_int, C.c_int, c_ip, C.c_void_p]
        L.orc_addr_set_neighb_ranks.argtypes = [C.c_void_p, c_ip]
        L.orc_gamg_npatchfaces.argtypes = [C.c_void_p, C.c_int]
        L.orc_gamg_free.argtypes = [C.c_void_p]
        L.orc_gamg_nlevels.argtypes = [C.c_void_p]
        L.orc_gamg_ncells.argtypes = [C.c_void_p, C.c_int]
        L.orc_gamg_nfaces.argtypes = [C.c_void_p, C.c_int]
        L.orc_gamg_restrict_addr.restype = c_ip
        L.orc_gamg_restrict_addr.argtypes = [C.c_void_p, C.c_int]
        L.orc_gamg_face_restrict_addr.restype = c_ip
        L.orc_gamg_face_restrict_addr.argtypes = [C.c_void_p, C.c_int]
        L.orc_gamg_face_flip.restype = C.POINTER(C.c_ubyte)
        L.orc_gamg_face_flip.argtypes = [C.c_void_p, C.c_int]
        L.orc_gamg_patch_face_restrict.restype = c_ip
        L.orc_gamg_patch_face_restrict.argtypes = [C.c_void_p, C.c_int]
        L.orc_gamg_agglomerate_patch_coeffs.argtypes = [C.c_void_p, C.c_int, c_dp, c_dp]
        L.orc_gamg_coarse_matrix.argtypes = [C.c_void_p, C.c_void_p, C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp]
        L.orc_gamg_set_coarsest_inverse.argtypes = [C.c_void_p, c_dp, c_ip, C.c_int]
        L.orc_gamg_set_scale_order.argtypes = [C.c_void_p, C.c_int]
        L.orc_addr_npatches.argtypes = [C.c_void_p]
        L.orc_set_reduce_hook.argtypes = [REDUCE_CB, C.c_void_p]
        L.orc_set_staged_ainv.argtypes = [C.c_int]
        for nm in ("orc_addr_patch_start", "orc_addr_face_cells"):
            getattr(L, nm).restype = c_ip
            getattr(L, nm).argtypes = [C.c_void_p]
        L.orc_sngrad.argtypes = [C.c_void_p, C.c_int, c_dp, c_dp, c_dp]
        L.orc_comm_sum.argtypes = [C.c_void_p, c_dp, C.c_int]
        L.orc_patch_neighbour_field.argtypes = [C.c_void_p, c_dp, C.c_void_p, c_dp]
        L.orc_gamg_addr.restype = C.c_void_p
        L.orc_gamg_addr.argtypes = [C.c_void_p, C.c_int]
        L.orc_gamg_solve.restype = C.c_int
        L.orc_gamg_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p, C.POINTER(Controls), c_dp, c_dp,
                                     C.c_void_p, C.POINTER(Perf), c_dp, C.c_int]
        L.orc_surface_integrate.argtypes = [C.c_void_p, C.c_int, c_dp, C.c_int, c_ip, c_dp, c_dp, c_dp,
                                            C.c_int, C.c_int]
        L.orc_gauss_grad.argtypes = [C.c_void_p, C.c_int, c_dp, c_dp, C.c_int, c_ip, c_dp, c_dp, c_dp, c_dp]
        L.orc_laplacian_fill.argtypes = [C.c_void_p, c_dp, c_dp, c_dp, c_dp]
        L.orc_convection_fill.argtypes = [C.c_void_p, c_dp, c_dp, c_dp, c_dp, c_dp]
        L.orc_interpolate_linear.argtypes = [C.c_void_p, C.c_int, c_dp, c_dp, c_dp]
        L.orc_add_boundary_diag.argtypes = [C.c_int, c_ip, c_dp, c_dp]
        L.orc_add_boundary_source.argtypes = [C.c_int, c_ip, c_dp, c_dp]
        L.orc_pcg_omp.restype = C.c_int
        L.orc_pcg_omp.argtypes = [C.c_void_p, C.c_int, C.POINTER(Controls), c_dp, c_dp, C.POINTER(Perf), C.c_int]
        L.orc_amul_omp.argtypes = [C.c_void_p, c_dp, c_dp, C.c_int]
        L.orc_pcg_stock_dic.restype = C.c_int
        L.orc_pcg_stock_dic.argtypes = [C.c_void_p, C.POINTER(Controls), c_dp, c_dp, C.POINTER(Perf)]
        L.orc_max_threads.restype = C.c_int
        _lib = L
    return _lib


def _d(a):
    return None if a is None else a.ctypes.data_as(c_dp)


def _i(a):
    return None if a is None else a.ctypes.data_as(c_ip)


def f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


def i32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.int32)


def controls(**kw):
    c = Controls()
    lib().orc_controls_default(C.byref(c))
    for k, v in kw.items():
        if not hasattr(c, k):
            raise KeyError(k)
        setattr(c, k, v)
    return c


class Addr:
    """lduAddressing (owner/neighbour + derived arrays + coupled patches)."""

    def __init__(self, nCells, lower, upper, patchStart=None, faceCells=None, _handle=None, neighbRank=None):
        self.nCells = int(nCells)
        self._own = _handle is None
        if _handle is not None:
            self.h = _handle
            self.nFaces = None
            return
        self.l = i32(lower)
        self.u = i32(upper)
        self.nFaces = len(self.l)
        self.patchStart = i32(patchStart) if patchStart is not None else None
        self.faceCells = i32(faceCells) if faceCells is not None else None
        nP = 0 if self.patchStart is None else len(self.patchStart) - 1
        self.nPatches = nP
        self.h = lib().orc_addr_create(self.nCells, self.nFaces, _i(self.l), _i(self.u), nP,
                                       _i(self.patchStart), _i(self.faceCells))
        if neighbRank is not None and nP:
            self.neighbRank = i32(neighbRank)
            lib().orc_addr_set_neighb_ranks(self.h, _i(self.neighbRank))

    def lower(self):
        return np.ctypeslib.as_array(lib().orc_addr_lower(self.h), (max(self.nFaces, 1),))[: self.nFaces].copy()

    def upper(self):
        return np.ctypeslib.as_array(lib().orc_addr_upper(self.h), (max(self.nFaces, 1),))[: self.nFaces].copy()

    def patch_start(self):
        nP = lib().orc_addr_npatches(self.h)
        if nP == 0:
            return np.zeros(0, np.int32)
        return np.ctypeslib.as_array(lib().orc_addr_patch_start(self.h), (nP + 1,)).copy()

    def face_cells(self):
        ps = self.patch_start()
        n = int(ps[-1]) if len(ps) else 0
        if n == 0:
            return np.zeros(0, np.int32)
        return np.ctypeslib.as_array(lib().orc_addr_face_cells(self.h), (n,)).copy()

    def patch_neighbour_field(self, psi, comm=None):
        """psi of the cell across every coupled patch face, flat over the patches"""
        ps = self.patch_start()
        n = int(ps[-1]) if len(ps) else 0
        out = np.zeros(max(n, 1))
        if n:
            lib().orc_patch_neighbour_field(self.h, _d(f64(psi)), _commp(comm), _d(out))
        return out[:n]

    def owner_start(self):
        return np.ctypeslib.as_array(lib().orc_addr_owner_start(self.h), (self.nCells + 1,)).copy()

    def losort(self):
        return np.ctypeslib.as_array(lib().orc_addr_losort(self.h), (max(self.nFaces, 1),))[: self.nFaces].copy()

    def losort_start(self):
        return np.ctypeslib.as_array(lib().orc_addr_losort_start(self.h), (self.nCells + 1,)).copy()

    def __del__(self):
        if getattr(self, "_own", False) and getattr(self, "h", None):
            lib().orc_addr_free(self.h)
            self.h = None


class PyComm:
    """Wraps python callables as an orc_comm:
    halo(send, patchStart) -> recv ; allsum(vals) -> vals ; gather(mine) -> (nRanks, n) array."""

    def __init__(self, halo=None, allsum=None, nCellsGlobal=0, gather=None, rank=0, nRanks=1):
        def _halo(ctx, send, recv, n, nP, pstart):
            s = np.ctypeslib.as_array(send, (n,))
            r = np.ctypeslib.as_array(recv, (n,))
            ps = np.ctypeslib.as_array(pstart, (nP + 1,)).copy()
            r[:] = halo(s.copy(), ps)

        def _sum(ctx, vals, n):
            v = np.ctypeslib.as_array(vals, (n,))
            v[:] = allsum(v.copy())

        def _gather(ctx, mine, n, allp):
            m = np.ctypeslib.as_array(mine, (n,))
            a = np.ctypeslib.as_array(allp, (nRanks * n,))
            a[:] = np.asarray(gather(m.copy())).reshape(-1)

        self._h = HALO_CB(_halo) if halo else HALO_CB()
        self._s = SUM_CB(_sum) if allsum else SUM_CB()
        self._g = GATHER_CB(_gather) if gather else GATHER_CB()
        self.c = Comm(None, self._h, self._s, int(nCellsGlobal), self._g, int(rank), int(nRanks))

    def ptr(self):
        return C.cast(C.byref(self.c), C.c_void_p)


def _commp(comm):
    return None if comm is None else comm.ptr()


class ReduceHook:
    """Lockstep with a device solve, for the calling thread while the block runs (single rank):
    fn(site, it, op, x, y, own) -> the value the oracle goes on with, at every global sum of the Krylov solvers,
    smoothSolver and normFactor.  site is a name of SITES, it the iteration body (0 for the sums before the first),
    op "sum" / "prod" / "mag" with the terms x[i], x[i]*y[i] or |x[i]|; x and y are views of the oracle's own
    vectors (y None unless op is "prod"), own is the oracle's sum.  staged_ainv: AINV with the device's association
    (orc_set_staged_ainv) for as long as the hook is armed."""

    def __init__(self, fn, staged_ainv=False):
        def _cb(ctx, site, it, op, x, y, n, own):
            xv = np.ctypeslib.as_array(x, (n,)) if n > 0 else np.zeros(0)
            yv = np.ctypeslib.as_array(y, (n,)) if (y and n > 0) else None
            return float(fn(SITES[site], it, RED_OPS[op], xv, yv, own))

        self._cb = REDUCE_CB(_cb)
        self.staged = bool(staged_ainv)

    def __enter__(self):
        lib().orc_set_reduce_hook(self._cb, None)
        lib().orc_set_staged_ainv(int(self.staged))
        return self

    def __exit__(self, *exc):
        lib().orc_set_reduce_hook(REDUCE_CB(), None)
        lib().orc_set_staged_ainv(0)


class Matrix:
    def __init__(self, addr, diag, upper, lower=None, bouCoeffs=None, intCoeffs=None):
        self.addr = addr
        self.diag, self.upper, self.lower = f64(diag), f64(upper), f64(lower)
        self.bou, self.intc = f64(bouCoeffs), f64(intCoeffs)
        self.h = lib().orc_matrix_create(addr.h, _d(self.diag), _d(self.upper), _d(self.lower),
                                         _d(self.bou), _d(self.intc))
        self.n = addr.nCells

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_matrix_free(self.h)
            self.h = None

    def _vec(self, n=None):
        return np.zeros(self.n if n is None else n)

    def amul(self, psi, comm=None):
        out = self._vec()
        lib().orc_amul(self.h, _d(f64(psi)), _d(out), _commp(comm))
        return out

    def tmul(self, psi, comm=None):
        out = self._vec()
        lib().orc_tmul(self.h, _d(f64(psi)), _d(out), _commp(comm))
        return out

    def sumA(self):
        out = self._vec()
        lib().orc_sumA(self.h, _d(out))
        return out

    def residual(self, psi, source, comm=None):
        out = self._vec()
        lib().orc_residual(self.h, _d(f64(psi)), _d(f64(source)), _d(out), _commp(comm))
        return out

    def H(self, psi):
        out = self._vec()
        lib().orc_H(self.h, _d(f64(psi)), _d(out))
        return out

    def H1(self):
        out = self._vec()
        lib().orc_H1(self.h, _d(out))
        return out

    def faceH(self, psi):
        out = self._vec(self.addr.nFaces)
        lib().orc_faceH(self.h, _d(f64(psi)), _d(out))
        return out

    def normFactor(self, psi, source, Apsi, comm=None):
        tmp = self._vec()
        return lib().orc_normFactor(self.h, _d(f64(psi)), _d(f64(source)), _d(f64(Apsi)), _d(tmp), _commp(comm))

    def precondition(self, kind, r, transpose=False):
        k = {"none": 0, "diagonal": 1, "AINV": 2, "DIC": 2, "DILU": 2}[kind]
        rD = 1.0 / self.diag
        w = self._vec()
        lib().orc_precondition(self.h, k, int(transpose), _d(rD), _d(f64(r)), _d(w))
        return w

    def jacobi(self, psi, source, nSweeps, omega=0.9, comm=None):
        p = f64(psi).copy()
        lib().orc_jacobi_smooth(self.h, omega, _d(p), _d(f64(source)), nSweeps, _commp(comm))
        return p

    def solve(self, solver, pre, psi0, source, comm=None, histCap=2048, **ctl):
        c = controls(**ctl)
        psi = f64(psi0).copy()
        hist = np.full(histCap, np.nan)
        perf = Perf()
        rc = lib().orc_solve(self.h, solver.encode(), (pre or "").encode(), C.byref(c), _d(psi),
                             _d(f64(source)), _commp(comm), C.byref(perf), _d(hist), histCap)
        if rc != 0:
            raise RuntimeError(f"orc_solve({solver},{pre}) failed rc={rc}")
        return psi, perf, hist[~np.isnan(hist)]

    def pcg_omp(self, pre, psi0, source, nThreads=None, **ctl):
        c = controls(**ctl)
        psi = f64(psi0).copy()
        perf = Perf()
        k = {"none": 0, "diagonal": 1, "AINV": 2, "DIC": 2, "DILU": 2}[pre]
        nT = nThreads or lib().orc_max_threads()
        lib().orc_pcg_omp(self.h, k, C.byref(c), _d(psi), _d(f64(source)), C.byref(perf), nT)
        return psi, perf

    def pcg_stock_dic(self, psi0, source, **ctl):
        """stock OpenFOAM numerics (true DIC + face-loop Amul), serial -- CPU baseline only"""
        c = controls(**ctl)
        psi = f64(psi0).copy()
        perf = Perf()
        lib().orc_pcg_stock_dic(self.h, C.byref(c), _d(psi), _d(f64(source)), C.byref(perf))
        return psi, perf

    def amul_omp(self, psi, nThreads=None):
        out = self._vec()
        lib().orc_amul_omp(self.h, _d(f64(psi)), _d(out), nThreads or lib().orc_max_threads())
        return out


class Gamg:
    """Pair agglomeration hierarchy (cached like the reference's MeshObject)."""

    def __init__(self, addr, faceWeights, nCellsInCoarsestLevel=10, mergeLevels=1, forward=None, comm=None):
        self.addr = addr
        self._fw = C.c_int(1 if forward is None else int(forward))
        w = f64(faceWeights)
        self.h = lib().orc_gamg_create(addr.h, _d(w), nCellsInCoarsestLevel, mergeLevels, C.byref(self._fw),
                                       _commp(comm))
        if not self.h:
            raise RuntimeError("orc_gamg_create failed (mergeLevels != 1?)")
        self.nLevels = lib().orc_gamg_nlevels(self.h)

    @property
    def forward(self):
        return self._fw.value

    def ncells(self, lev):
        return lib().orc_gamg_ncells(self.h, lev)

    def nfaces(self, lev):
        return lib().orc_gamg_nfaces(self.h, lev)

    def npatchfaces(self, lev):
        return lib().orc_gamg_npatchfaces(self.h, lev)

    def restrict_addr(self, lev):
        n = self.addr.nCells if lev == 0 else self.ncells(lev - 1)
        return np.ctypeslib.as_array(lib().orc_gamg_restrict_addr(self.h, lev), (n,)).copy()

    def face_restrict_addr(self, lev):
        n = self.addr.nFaces if lev == 0 else self.nfaces(lev - 1)
        return np.ctypeslib.as_array(lib().orc_gamg_face_restrict_addr(self.h, lev), (max(n, 1),))[:n].copy()

    def face_flip(self, lev):
        n = self.addr.nFaces if lev == 0 else self.nfaces(lev - 1)
        return np.ctypeslib.as_array(lib().orc_gamg_face_flip(self.h, lev), (max(n, 1),))[:n].copy()

    def patch_face_restrict(self, lev):
        """fine coupled-patch face (flat over the patches of level lev's fine side) -> coarse patch face (flat)"""
        fine = self.addr if lev == 0 else self.level_addr(lev - 1)
        ps = fine.patch_start()
        n = int(ps[-1]) if len(ps) else 0
        if n == 0:
            return np.zeros(0, np.int32)
        return np.ctypeslib.as_array(lib().orc_gamg_patch_face_restrict(self.h, lev), (n,)).copy()

    def agglomerate_patch_coeffs(self, lev, fine):
        out = np.zeros(max(self.npatchfaces(lev), 1))
        lib().orc_gamg_agglomerate_patch_coeffs(self.h, lev, _d(f64(fine)), _d(out))
        return out[: self.npatchfaces(lev)]

    def coarse_matrix(self, matrix, lev):
        """dict(diag, upper, lower, bou, int) of coarse level lev for the finest `matrix`, as the solve builds it
        (lower None for a symmetric matrix)"""
        n, nf, npf = self.ncells(lev), self.nfaces(lev), self.npatchfaces(lev)
        d, u, lo, b, i = (np.zeros(max(k, 1)) for k in (n, nf, nf, npf, npf))
        lib().orc_gamg_coarse_matrix(matrix.h, self.h, lev, _d(d), _d(u), _d(lo), _d(b), _d(i))
        return dict(diag=d[:n], upper=u[:nf], lower=None if matrix.lower is None else lo[:nf], bou=b[:npf], int=i[:npf])

    def set_coarsest_inverse(self, inv=None, perm=None):
        """Solve the coarsest level with the given rows of an inverse (this rank's banded rows x N global banded
        columns) and banded permutation, one FMA chain per row as the device applies it; None: the LU again."""
        if inv is None:
            lib().orc_gamg_set_coarsest_inverse(self.h, None, None, 0)
            return
        inv = f64(inv)
        self._inv = (inv, i32(perm))
        lib().orc_gamg_set_coarsest_inverse(self.h, _d(inv), _i(self._inv[1]), inv.shape[1])

    def set_scale_order(self, descending):
        lib().orc_gamg_set_scale_order(self.h, int(bool(descending)))

    def level_addr(self, lev):
        a = Addr(self.ncells(lev), None, None, _handle=lib().orc_gamg_addr(self.h, lev))
        a.nFaces = self.nfaces(lev)
        return a

    def solve(self, matrix, smoother, psi0, source, histCap=2048, comm=None, **ctl):
        c = controls(**ctl)
        psi = f64(psi0).copy()
        hist = np.full(histCap, np.nan)
        perf = Perf()
        rc = lib().orc_gamg_solve(matrix.h, self.h, (smoother or "").encode(), C.byref(c), _d(psi),
                                  _d(f64(source)), _commp(comm), C.byref(perf), _d(hist), histCap)
        if rc != 0:
            raise RuntimeError(f"orc_gamg_solve failed rc={rc}")
        return psi, perf, hist[~np.isnan(hist)]

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_gamg_free(self.h)
            self.h = None


# ---- finite-volume face sums ----

def surface_integrate(addr, ssf, bFaceCells, bssf, V, nComp=1, divideByV=True, neiSign=-1):
    out = np.zeros(addr.nCells * nComp)
    bfc = i32(bFaceCells)
    lib().orc_surface_integrate(addr.h, nComp, _d(f64(ssf)), len(bfc), _i(bfc), _d(f64(bssf)), _d(f64(V)),
                                _d(out), int(divideByV), neiSign)
    return out.reshape(addr.nCells, nComp) if nComp > 1 else out


def gauss_grad(addr, Sf, ssf, bFaceCells, bSf, bssf, V, nComp=1):
    out = np.zeros(addr.nCells * 3 * nComp)
    bfc = i32(bFaceCells)
    lib().orc_gauss_grad(addr.h, nComp, _d(f64(Sf)), _d(f64(ssf)), len(bfc), _i(bfc), _d(f64(bSf)),
                         _d(f64(bssf)), _d(f64(V)), _d(out))
    return out.reshape(addr.nCells, 3 * nComp)


def laplacian_fill(addr, deltaCoeffs, gammaMagSf):
    upper = np.zeros(addr.nFaces)
    diag = np.zeros(addr.nCells)
    lib().orc_laplacian_fill(addr.h, _d(f64(deltaCoeffs)), _d(f64(gammaMagSf)), _d(upper), _d(diag))
    return upper, diag


def convection_fill(addr, weights, phi):
    lower = np.zeros(addr.nFaces)
    upper = np.zeros(addr.nFaces)
    diag = np.zeros(addr.nCells)
    lib().orc_convection_fill(addr.h, _d(f64(weights)), _d(f64(phi)), _d(lower), _d(upper), _d(diag))
    return lower, upper, diag


def sngrad(addr, deltaCoeffs, vf, nComp=1):
    """snGradScheme::snGrad on the internal faces: deltaCoeffs*(vf[nei] - vf[own])"""
    out = np.zeros(addr.nFaces * nComp)
    lib().orc_sngrad(addr.h, nComp, _d(f64(deltaCoeffs)), _d(f64(vf)), _d(out))
    return out.reshape(addr.nFaces, nComp) if nComp > 1 else out


def interpolate_linear(addr, w, vf, nComp=1):
    sf = np.zeros(addr.nFaces * nComp)
    lib().orc_interpolate_linear(addr.h, nComp, _d(f64(w)), _d(f64(vf)), _d(sf))
    return sf.reshape(addr.nFaces, nComp) if nComp > 1 else sf


def add_boundary_diag(bFaceCells, internalCoeffs, diag):
    d = f64(diag).copy()
    bfc = i32(bFaceCells)
    lib().orc_add_boundary_diag(len(bfc), _i(bfc), _d(f64(internalCoeffs)), _d(d))
    return d


def add_boundary_source(bFaceCells, boundaryCoeffs, source):
    s = f64(source).copy()
    bfc = i32(bFaceCells)
    lib().orc_add_boundary_source(len(bfc), _i(bfc), _d(f64(boundaryCoeffs)), _d(s))
    return s


def max_threads():
    return lib().orc_max_threads()
