"""Dry-run aid for the GPU tests (NOT part of the product and not used by default): an object with the
surface of rapidcfd-dev_b200.capi backed by the CPU oracle and CPU torch tensors.

    B200LDU_DRYRUN_ORACLE=1 python -m pytest tests/test_ref_golden.py tests/test_zz_golden.py tests/test_zzz_fvm_gpu.py -m gpu -q

runs the `-m gpu` tests of those files with this stand-in instead of the CUDA library: it checks the
tests' own logic (indexing of the fixtures, shapes, iteration windows, tolerances) where no GPU is
available.  It says nothing about the CUDA path; on a GPU box the variable is unset and the real library
is used."""
import numpy as np

from oracle import fvm_oracle as fo
from oracle import ldu_oracle as orc


class _Ctx:
    device = "cpu"

    def __init__(self, comm=None):
        self.comm = comm       # orc.PyComm of this rank (multi-rank dry runs), None on a single domain

    def close(self):
        pass


class LduAddressing:
    def __init__(self, ctx, nCells, lower, upper, patchStart=None, faceCells=None, neighbRank=None, cellCentres=None):
        self.ctx = ctx
        self.nPatchFaces = 0 if patchStart is None else int(patchStart[-1])
        self.nCells, self.nFaces = int(nCells), len(lower)
        self.o = orc.Addr(nCells, lower, upper) if patchStart is None else orc.Addr(nCells, lower, upper, patchStart,
                                                                                     faceCells, neighbRank=neighbRank)

    def close(self):
        pass


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


class LduMatrix:
    def __init__(self, addr):
        self.addr = addr
        self.m = None

    def set(self, diag, upper, lower=None, bou=None, intc=None):
        self.m = orc.Matrix(self.addr.o, _np(diag), _np(upper), _np(lower), _np(bou), _np(intc))
        # the library copies the coefficients (b200ldu_matrix_set): a later change of the caller's arrays -- fvMatrix::relax,
        # setReference -- does not reach A / H / flux / residual / solve until the matrix is set again
        self.coeffs = tuple(None if x is None else x.clone() for x in (diag, upper, lower, bou, intc))
        return self

    def _t(self, a):
        import torch
        return torch.from_numpy(np.ascontiguousarray(a))

    def Amul(self, x):
        return self._t(self.m.amul(_np(x)))

    def Tmul(self, x):
        return self._t(self.m.tmul(_np(x)))

    def sumA(self, like):
        return self._t(self.m.sumA())

    def residual(self, x, b):
        return self._t(self.m.residual(_np(x), _np(b)))

    def H(self, x):
        return self._t(self.m.H(_np(x)))

    def H1(self, like):
        return self._t(self.m.H1())

    def faceH(self, x):
        return self._t(self.m.faceH(_np(x)))

    def precondition(self, name, r, transpose=False):
        return self._t(self.m.precondition(name, _np(r), transpose))

    def smooth(self, name, x, b, nSweeps, omega=0.9):
        return self._t(self.m.jacobi(_np(x), _np(b), nSweeps, omega=omega))

    def solve(self, solver, pre, psi, source, gamg=None, histCap=0, **ctl):
        if solver == "GAMG":
            out, perf, hist = gamg.o.solve(self.m, pre, _np(psi), _np(source), comm=self.addr.ctx.comm, **ctl)
        else:
            out, perf, hist = self.m.solve(solver, pre, _np(psi), _np(source), comm=self.addr.ctx.comm, **ctl)
        psi.copy_(self._t(out))
        return perf, (hist if histCap else hist[:0])

    def close(self):
        pass


class FvMatrix:
    """surface of capi.FvMatrix over oracle/fvm_oracle.py (dry runs of tests/test_zzz_fvm_gpu.py)"""

    def __init__(self, matrix, nComp, diag, source, psi, V, internalCoeffs=None, boundaryCoeffs=None):
        self.m, self.nc = matrix, int(nComp)
        self.diag, self.source, self.psi, self.V, self.ic, self.bc = diag, source, psi, V, internalCoeffs, boundaryCoeffs

    def _o(self, diag=None, source=None):
        own, upper, lower, bou, intc = self.m.coeffs
        a = self.m.addr
        return fo.FvMatrix(orc, a.o, self.nc, _np(own if diag is None else diag), _np(upper), _np(lower),
                           _np(self.source if source is None else source), _np(self.psi), _np(self.V), a.bfc,
                           _np(self.ic), _np(self.bc), couInt=_np(intc), couBou=_np(bou), comm=a.ctx.comm)

    def _t(self, a):
        import torch
        return torch.from_numpy(np.ascontiguousarray(a).ravel())

    def _pnf(self, pnf):
        return None if pnf is None else _np(pnf).reshape(-1, self.nc)

    def addBoundaryDiag(self, diag, cmpt):
        d = _np(diag).copy()
        self._o().addBoundaryDiag(d, cmpt)
        diag.copy_(self._t(d))

    def addCmptAvBoundaryDiag(self, diag):
        d = _np(diag).copy()
        self._o().addCmptAvBoundaryDiag(d)
        diag.copy_(self._t(d))

    def addBoundarySource(self, source, pnf=None):
        s = _np(source).reshape(-1, self.nc).copy()
        self._o().addBoundarySource(s, pnf is not None, self._pnf(pnf))
        source.copy_(self._t(s))

    def A(self):
        return self._t(self._o().A())

    def H(self, pnf=None):
        return self._t(self._o().H(pnf=self._pnf(pnf)))

    def flux(self, nBFaces, nCoupledFaces=0, pnf=None):
        return tuple(self._t(x) for x in self._o().flux(self._pnf(pnf)))

    def residual(self, pnf=None):
        return self._t(self._o().residual(self._pnf(pnf)))

    def relax(self, alpha):
        o = self._o(diag=self.diag)            # b200ldu_fvm_relax works on the caller's diag / source
        o.relax(alpha)
        self.diag.copy_(self._t(o.diag))
        self.source.copy_(self._t(o.source))

    def setReference(self, celli, value):
        """source[celli] += diag[celli]*value; diag[celli] *= 2 (fvMatrix.C:965-983): in place on the caller's arrays,
        before the matrix copies them (LduMatrix.set) -- touches no coefficient of the matrix itself"""
        if celli < 0:
            return
        v = np.atleast_1d(np.asarray(value, np.float64))
        d, s = _np(self.diag).copy(), _np(self.source).reshape(-1, self.nc).copy()
        s[celli] += d[celli] * v
        d[celli] += d[celli]
        self.diag.copy_(self._t(d))
        self.source.copy_(self._t(s))

    def solve(self, solver, pre, gamg=None, pnf=None, **ctl):
        psi, perfs, _ = self._o().solve(solver, pre, gamg.o if gamg is not None else None, self._pnf(pnf), **ctl)
        self.psi.copy_(self._t(psi))
        return perfs


class FieldOps:
    """surface of capi.FieldOps in numpy (one rounded operation per call, like the device kernels)"""

    def __init__(self, ctx):
        self.ctx = ctx

    @staticmethod
    def _t(a):
        import torch
        return torch.from_numpy(np.ascontiguousarray(a).ravel())

    def _bin(self, f, a, b, nca, ncb):
        A, B = _np(a).reshape(-1, nca), _np(b).reshape(-1, ncb)
        return self._t(f(A, B))

    def add(self, a, b, nca=1, ncb=1):
        return self._bin(np.add, a, b, nca, ncb)

    def sub(self, a, b, nca=1, ncb=1):
        return self._bin(np.subtract, a, b, nca, ncb)

    def mul(self, a, b, nca=1, ncb=1):
        return self._bin(np.multiply, a, b, nca, ncb)

    def div(self, a, b, nca=1, ncb=1):
        return self._bin(np.divide, a, b, nca, ncb)

    def neg(self, a):
        return self._t(-_np(a))

    def mag(self, a):
        return self._t(np.abs(_np(a)))

    def smul(self, s, a):
        return self._t(s * _np(a))

    def rdiv(self, s, a):
        return self._t(s / _np(a))

    def sadd(self, a, s):
        return self._t(_np(a) + s)

    def rsub(self, s, a):
        return self._t(s - _np(a))

    def smin(self, a, s):
        return self._t(fo.min_(_np(a), s))

    def sdiv(self, a, s):
        return self._t(_np(a) / s)

    def smax(self, a, s):
        return self._t(fo.max_(_np(a), s))

    def pos(self, a):
        return self._t(np.where(_np(a) >= 0, 1.0, 0.0))

    def bmax(self, a, b):
        return self._t(fo.max_(_np(a), _np(b)))

    def symm_magsqr(self, T):
        from oracle import kepsilon_oracle as ko
        return self._t(ko.symm_magsqr(_np(T).reshape(-1, 9)))

    def dot3(self, a, b):
        A, B = _np(a).reshape(-1, 3), _np(b).reshape(-1, 3)
        return self._t((A[:, 0] * B[:, 0] + A[:, 1] * B[:, 1]) + A[:, 2] * B[:, 2])

    def gather(self, cells, f, nc=1):
        return self._t(_np(f).reshape(-1, nc)[_np(cells)])


class GamgAgglomeration:
    def __init__(self, addr, faceWeights, nCellsInCoarsestLevel=10, mergeLevels=1, forward=1):
        self.o = orc.Gamg(addr.o, faceWeights, nCellsInCoarsestLevel, mergeLevels=mergeLevels, forward=forward)
        self.nLevels = self.o.nLevels

    @property
    def forward(self):
        return self.o.forward

    def level_size(self, lev):
        return self.o.ncells(lev), self.o.nfaces(lev)

    def restrict_addr(self, lev):
        return self.o.restrict_addr(lev)

    def close(self):
        pass


class _Capi:
    LduAddressing = LduAddressing
    LduMatrix = LduMatrix
    FvMatrix = FvMatrix
    FieldOps = FieldOps

    @staticmethod
    def fv_patch_neighbour_field(addr, nc, field):
        f = _np(field).reshape(-1, nc)
        cols = [addr.o.patch_neighbour_field(np.ascontiguousarray(f[:, k]), addr.ctx.comm) for k in range(nc)]
        return FieldOps._t(np.stack(cols, axis=1))

    @staticmethod
    def fv_sngrad(addr, nc, delta, vf):
        return FieldOps._t(orc.sngrad(addr.o, _np(delta), _np(vf), nc))

    @staticmethod
    def fv_convection_fill(addr, w, phi):
        return tuple(FieldOps._t(x) for x in orc.convection_fill(addr.o, _np(w), _np(phi)))

    @staticmethod
    def fv_laplacian_fill(addr, delta, g):
        return tuple(FieldOps._t(x) for x in orc.laplacian_fill(addr.o, _np(delta), _np(g)))

    @staticmethod
    def fv_interpolate_linear(addr, nc, w, vf):
        return FieldOps._t(orc.interpolate_linear(addr.o, _np(w), _np(vf), nc))

    @staticmethod
    def fv_flux_linear(addr, Sf, w, U):
        Uf = np.asarray(orc.interpolate_linear(addr.o, _np(w), _np(U), 3)).reshape(-1, 3)
        S = _np(Sf).reshape(-1, 3)
        return FieldOps._t((S[:, 0] * Uf[:, 0] + S[:, 1] * Uf[:, 1]) + S[:, 2] * Uf[:, 2])

    @staticmethod
    def fv_grad_linear(addr, nc, Sf, w, vf, bSf, bvf, V):
        sf = orc.interpolate_linear(addr.o, _np(w), _np(vf), nc)
        return FieldOps._t(orc.gauss_grad(addr.o, _np(Sf), np.asarray(sf).ravel(), addr.bfc, _np(bSf), _np(bvf), _np(V), nc))

    @staticmethod
    def fv_surface_integrate(addr, nc, ssf, bssf, V, divideByV=True, neiSign=-1):
        return FieldOps._t(orc.surface_integrate(addr.o, _np(ssf), addr.bfc, _np(bssf), _np(V), nc, divideByV, neiSign))

    @staticmethod
    def fv_limited_weights(ctx, faceFlux, limiter=None, cdWeights=None):
        from oracle import limiters_oracle as lo
        import torch
        w = lo.limited_weights(_np(faceFlux), None if limiter is None else _np(limiter), None if cdWeights is None else _np(cdWeights))
        return torch.from_numpy(np.ascontiguousarray(w))

    @staticmethod
    def mules_limiter(addr, V, rDeltaT, psi, psi0, psiB, phiBD, phiBDB, phiCorr, phiCorrB, psiMax, psiMin, nLimiterIter=3,
                      rho=None, rho0=None, Sp=None, Su=None, nCoupled=0):
        from oracle import mules_oracle as mo
        assert not nCoupled, "the stand-in runs single-domain MULES only (decomposed: oracle.mules_oracle.limiter_ranks)"
        o = lambda x: None if x is None else _np(x)
        lam, lamB = mo.limiter(addr.o.nCells, addr.o.lower(), addr.o.upper(), addr.bfc, _np(V), rDeltaT, _np(psi), _np(psi0), _np(psiB),
                               _np(phiBD), _np(phiBDB), _np(phiCorr), _np(phiCorrB), psiMax, psiMin, nLimiterIter, o(rho), o(rho0),
                               o(Sp), o(Su))
        return FieldOps._t(lam), FieldOps._t(lamB)

    @staticmethod
    def mules_limiter_corr(addr, V, rDeltaT, psi, psiB, phiB, phiCorr, phiCorrB, psiMax, psiMin, nLimiterIter=3, rho=None, Sp=None,
                           Su=None, extremaCoeff=0.0, nCoupled=0):
        from oracle import mules_oracle as mo
        assert not nCoupled, "the stand-in runs single-domain MULES only"
        o = lambda x: None if x is None else _np(x)
        lam, lamB = mo.limiter(addr.o.nCells, addr.o.lower(), addr.o.upper(), addr.bfc, _np(V), rDeltaT, _np(psi), _np(psi), _np(psiB),
                               np.zeros(addr.nFaces), _np(phiB), _np(phiCorr), _np(phiCorrB), psiMax, psiMin, nLimiterIter, o(rho), None,
                               o(Sp), o(Su), corr=True, extremaCoeff=extremaCoeff)
        return FieldOps._t(lam), FieldOps._t(lamB)

    @staticmethod
    def fv_boundary_set(addr, bFaceCells):
        addr.bfc = np.asarray(bFaceCells, np.int32).copy()
    GamgAgglomeration = GamgAgglomeration

    @staticmethod
    def Context(dev):
        return _Ctx()

    @staticmethod
    def mesh_to_device(ctx, mesh, with_centres=True):
        ps, fc = mesh.patch_start_facecells()
        nr = [p.neighbRank for p in mesh.coupled_patches()]
        if not nr:
            return LduAddressing(ctx, mesh.nCells, mesh.lower, mesh.upper)
        return LduAddressing(ctx, mesh.nCells, mesh.lower, mesh.upper, ps, fc, nr)

    @staticmethod
    def polymesh_to_device(ctx, pm, cellCentres=None):
        lo, up = pm.ldu()
        ps, fc, nr = pm.coupled_interface_arrays()
        return LduAddressing(ctx, pm.nCells, lo, up, ps, fc, nr)


def fixture():
    """what the `gpu` fixtures yield: (capi, ctx, torch)"""
    import torch
    return _Capi, _Ctx(), torch
