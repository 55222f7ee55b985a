"""CPU restatement of the fvMatrix glue around the linear solvers (SURVEY.md section 8, row a17) -- TEST
INFRASTRUCTURE ONLY, like the rest of oracle/.  numpy compositions of the C oracle's primitives; numpy rounds
every elementwise operation separately (no contraction) and np.add.at / np.subtract.at accumulate sequentially
in index order, which is the order of the reference's per-patch functors (ascending patch face per cell,
patches in mesh order).  PINNED to the reference's own source: fvMatrix.H / fvMatrix.C / fvMatrixSolve.C /
fvScalarMatrix.C compile for the host against oracle/ref_harness/shim_fvm/ (fields, GeometricField, fvMesh and
lduMatrix reduced to what the exercised members touch; the linear solver behind solveSegregated records the
diagonal and source it is handed) and tests/test_reference_functors.py compares, bit for bit, for scalar and
vector fields with and without coupled patches: addBoundaryDiag / addCmptAvBoundaryDiag / addBoundarySource,
setReference, relax, D, A, H, flux and residual (scalar), and what solveSegregated passes to the solver per
component.  tests/test_oracle_fvm.py adds dense-matrix algebra and decomposed-case checks.

Paths: FV/ = /root/reference/src/finiteVolume/.

Boundary model: the non-coupled boundary faces of all patches as one flat list in patch order (face cell,
internalCoeffs, boundaryCoeffs per face and component); coupled (processor / cyclic) patches are those of the
addressing, their coefficients the matrix' interfaceIntCoeffs / interfaceBouCoeffs -- one scalar per face,
used for every component (what processorFvPatchField produces for vectors, coupledFvPatchField.C:116-176).
Fields with nc components are (n, nc) arrays.

Findings while restating (mirrored, not corrected; both reproduced by running the reference's code):
 * fvMatrix<Type>::H (fvMatrix.C:1458-1485) fills Hphi with boundaryDiagCmpt*psi and then calls the two-argument
   lduMatrix::H(Hphi, psi), which starts with Hpsi = 0 (lduMatrixTemplates.C:53): the boundary-diagonal term of
   stock OpenFOAM is lost.  It vanishes anyway when internalCoeffs are equal in all components (fixedValue,
   zeroGradient); `boundaryDiagInH=True` restores the stock term.
 * fvMatrix<scalar>::residual (fvScalarMatrix.C:195-240) counts the neighbour term of coupled patches twice:
   lduMatrix::residual applies the interfaces and addBoundarySource(res) adds boundaryCoeffs*patchNeighbourField
   again (`couples` defaults to true) -- stock OpenFOAM 2.3 has the same lines.
"""
import numpy as np


def max_(s1, s2):
    """max of two scalars as the reference defines it (label.H:285-297, instantiated for doubles by doubleFloat.H:69-86):
    (s1 > s2) ? s1 : s2 -- the second operand on a tie (max(+0, -0) = -0) and whenever either operand is NaN"""
    s1, s2 = np.asarray(s1, float), np.asarray(s2, float)
    return np.where(s1 > s2, s1, s2)


def min_(s1, s2):
    """(s1 < s2) ? s1 : s2, the reference's min (label.H:285-297)"""
    s1, s2 = np.asarray(s1, float), np.asarray(s2, float)
    return np.where(s1 < s2, s1, s2)


def _cmptAv(ic):            # VectorSpaceI.H:428-447: ((x + y) + z)/3; a scalar is its own average
    if ic.shape[1] == 1:
        return ic[:, 0].copy()
    s = ic[:, 0].copy()
    for k in range(1, ic.shape[1]):
        s = s + ic[:, k]
    return s / ic.shape[1]


class FvMatrix:
    """fvMatrix<Type> (FV/fvMatrices/fvMatrix/fvMatrix.H) for Type = scalar (nc 1) or vector (nc 3)."""

    def __init__(self, orc, addr, nc, diag, upper, lower, source, psi, V, bFaceCells=None, internalCoeffs=None,
                 boundaryCoeffs=None, couInt=None, couBou=None, comm=None):
        self.orc, self.addr, self.nc, self.comm = orc, addr, int(nc), comm
        self.n = addr.nCells
        self.diag = np.array(diag, float)
        self.upper = np.array(upper, float)
        self.lower = None if lower is None else np.array(lower, float)
        self.source = np.array(source, float).reshape(self.n, self.nc)
        self.psi = np.array(psi, float).reshape(self.n, self.nc)
        self.V = np.array(V, float)
        self.bfc = np.zeros(0, np.int64) if bFaceCells is None else np.asarray(bFaceCells, np.int64)
        nB = len(self.bfc)
        self.ic = np.zeros((nB, self.nc)) if internalCoeffs is None else np.array(internalCoeffs, float).reshape(nB, self.nc)
        self.bc = np.zeros((nB, self.nc)) if boundaryCoeffs is None else np.array(boundaryCoeffs, float).reshape(nB, self.nc)
        self.cfc = np.asarray(addr.face_cells(), np.int64)           # coupled patch faces, flat
        nC = len(self.cfc)
        self.couInt = np.zeros(nC) if couInt is None else np.array(couInt, float)
        self.couBou = np.zeros(nC) if couBou is None else np.array(couBou, float)

    # ---- helpers -------------------------------------------------------------------------------------
    def _ldu(self, diag=None):
        return self.orc.Matrix(self.addr, self.diag if diag is None else diag, self.upper, self.lower,
                               self.couBou if len(self.cfc) else None, self.couInt if len(self.cfc) else None)

    def patchNeighbourField(self, psi=None):
        """coupledFvPatchField::patchNeighbourField of every coupled face, (nCoupledFaces, nc)"""
        psi = self.psi if psi is None else psi
        if not len(self.cfc):
            return np.zeros((0, self.nc))
        return np.stack([self.addr.patch_neighbour_field(np.ascontiguousarray(psi[:, k]), self.comm)
                         for k in range(self.nc)], axis=1)

    # ---- fvMatrix.C:209-243 ---------------------------------------------------------------------------
    def addBoundaryDiag(self, diag, cmpt):
        """diag[cell] += internalCoeffs.component(cmpt) over EVERY patch, coupled ones included (:209-226)"""
        np.add.at(diag, self.bfc, self.ic[:, cmpt])
        np.add.at(diag, self.cfc, self.couInt)

    def addCmptAvBoundaryDiag(self, diag):
        """:230-243; a coupled patch of a vector field holds (c, c, c), whose average ((c + c) + c)/3 is not always c"""
        np.add.at(diag, self.bfc, _cmptAv(self.ic))
        np.add.at(diag, self.cfc, _cmptAv(np.repeat(self.couInt[:, None], self.nc, axis=1)))

    # ---- fvMatrix.C:290-348 ---------------------------------------------------------------------------
    def addBoundarySource(self, source, couples=True, pnf=None):
        """non-coupled patches add boundaryCoeffs; coupled ones cmptMultiply(boundaryCoeffs, patchNeighbourField)
        when `couples` (products rounded, then added: fvMatrixAddBoundarySourceFunctor :246-286)"""
        for k in range(self.nc):
            np.add.at(source[:, k], self.bfc, self.bc[:, k])
        if couples and len(self.cfc):
            pnf = self.patchNeighbourField() if pnf is None else pnf
            for k in range(self.nc):
                np.add.at(source[:, k], self.cfc, self.couBou * pnf[:, k])

    # ---- fvMatrix.C:965-983 ---------------------------------------------------------------------------
    def setReference(self, celli, value):
        """source[celli] += diag[celli]*value; diag[celli] = 2*diag[celli]"""
        if celli >= 0:
            self.source[celli] = self.source[celli] + self.diag[celli] * np.atleast_1d(np.asarray(value, float))
            self.diag[celli] = 2 * self.diag[celli]

    # ---- fvMatrix.C:1088-1345 -------------------------------------------------------------------------
    def relax(self, alpha):
        if alpha <= 0:
            return
        D, S = self.diag, self.source
        D0 = D.copy()
        sumOff = np.zeros(self.n)
        self.orc.lib().orc_sumMagOffDiag(self.addr.h, self.orc._d(self.upper),
                                         self.orc._d(self.lower if self.lower is not None else self.upper),
                                         self.orc._d(sumOff))
        # non-coupled patches: the largest |component| of the internal coefficient (:1197-1218)
        np.add.at(D, self.bfc, np.abs(self.ic).max(axis=1))
        # coupled patches: component 0 into the diagonal, |boundary coefficient| into the off-diagonal sum (:1152-1194)
        np.add.at(D, self.cfc, self.couInt)
        np.add.at(sumOff, self.cfc, np.abs(self.couBou))
        D[:] = np.maximum(np.abs(D), sumOff)        # :1279-1280
        D[:] = D / alpha                            # :1283
        np.add.at(D, self.bfc, -self.ic.min(axis=1))   # :1317-1336  (-cmptMin)
        np.add.at(D, self.cfc, -self.couInt)           # :1299-1314
        S[:] = S + (D - D0)[:, None] * self.psi     # :1344

    # ---- fvMatrix.C:1375-1455 -------------------------------------------------------------------------
    def D(self):
        d = self.diag.copy()
        self.addCmptAvBoundaryDiag(d)
        return d

    def A(self):
        """A = D()/V (:1425-1430)"""
        return self.D() / self.V

    # ---- fvMatrix.C:1458-1508, fvScalarMatrix.C:252-283 -----------------------------------------------
    def H(self, boundaryDiagInH=False, pnf=None):
        M = self._ldu()
        H = np.stack([M.H(np.ascontiguousarray(self.psi[:, k])) for k in range(self.nc)], axis=1)
        if boundaryDiagInH and self.nc > 1:   # stock OpenFOAM: Hphi = boundaryDiagCmpt*psi + lduMatrix::H(psi)
            for k in range(self.nc):
                bd = np.zeros(self.n)
                self.addBoundaryDiag(bd, k)
                bd = -bd
                self.addCmptAvBoundaryDiag(bd)
                H[:, k] = bd * self.psi[:, k] + H[:, k]
        H = H + self.source
        self.addBoundarySource(H, True, pnf)
        return H / self.V[:, None]

    # ---- fvMatrix.C:1591-1660 -------------------------------------------------------------------------
    def flux(self, pnf=None):
        """returns (internal faces (nFaces, nc), non-coupled boundary faces (nB, nc), coupled faces (nC, nc))"""
        M = self._ldu()
        internal = np.stack([M.faceH(np.ascontiguousarray(self.psi[:, k])) for k in range(self.nc)], axis=1)
        boundary = self.ic * self.psi[self.bfc] - self.bc
        if len(self.cfc):
            pnf = self.patchNeighbourField() if pnf is None else pnf
            coupled = self.couInt[:, None] * self.psi[self.cfc] - self.couBou[:, None] * pnf
        else:
            coupled = np.zeros((0, self.nc))
        return internal, boundary, coupled

    # ---- fvScalarMatrix.C:195-240 ---------------------------------------------------------------------
    def residual(self, pnf=None):
        assert self.nc == 1
        bd = np.zeros(self.n)
        self.addBoundaryDiag(bd, 0)
        src = self.source[:, 0] - bd * self.psi[:, 0]        # fvScalarMatrixResidualFunctor
        res = self._ldu().residual(self.psi[:, 0], src, self.comm)[:, None]
        self.addBoundarySource(res, True, pnf)
        return res[:, 0]

    # ---- fvScalarMatrix.C:142-192, fvMatrixSolve.C:104-226 --------------------------------------------
    def solve(self, solver, precond, gamg=None, pnf=None, **controls):
        """solveSegregated.  Returns (psi, [perf per component], [residual history per component])."""
        psi = self.psi.copy()
        perfs, hists = [], []
        if self.nc == 1:
            diag = self.diag.copy()
            self.addBoundaryDiag(diag, 0)
            total = self.source.copy()
            self.addBoundarySource(total, False)
            p, perf, hist = self._solve(diag, psi[:, 0], total[:, 0], solver, precond, gamg, controls)
            psi[:, 0] = p
            return psi, [perf], [hist]
        source = self.source.copy()
        pnf = (self.patchNeighbourField() if pnf is None else pnf) if len(self.cfc) else None
        self.addBoundarySource(source, True, pnf)               # coupled part included here (:130-133) ...
        for k in range(self.nc):
            diag = self.diag.copy()
            self.addBoundaryDiag(diag, k)
            sk = np.ascontiguousarray(source[:, k])
            if pnf is not None:                                 # ... and taken out again through
                np.subtract.at(sk, self.cfc, self.couBou * pnf[:, k])   # updateMatrixInterfaces (:170-186)
            p, perf, hist = self._solve(diag, np.ascontiguousarray(psi[:, k]), sk, solver, precond, gamg, controls)
            psi[:, k] = p
            perfs.append(perf)
            hists.append(hist)
        return psi, perfs, hists

    def _solve(self, diag, psi0, source, solver, precond, gamg, controls):
        M = self._ldu(diag)
        if solver == "GAMG":
            return gamg.solve(M, precond, psi0, source, comm=self.comm, **controls)
        return M.solve(solver, precond, psi0, source, comm=self.comm, **controls)


# ---- boundary-condition coefficients the schemes hand to the matrix ------------------------------------
def fixedValue_laplacian_coeffs(gammaMagSf_b, deltaCoeffs_b, value):
    """internalCoeffs / boundaryCoeffs of fvm::laplacian on a fixedValue patch: gaussLaplacianScheme.C:66-86 with
    fixedValueFvPatchField.C:136-146: internalCoeffs = pGamma*(-1*delta), boundaryCoeffs = -pGamma*(delta*value)."""
    value = np.atleast_2d(np.asarray(value, float))
    g = np.asarray(gammaMagSf_b, float)[:, None]
    d = np.asarray(deltaCoeffs_b, float)[:, None]
    return g * (-d) * np.ones_like(value), (-g) * (d * value)


def zeroGradient_coeffs(nB, nc):
    """zeroGradientFvPatchField.C: gradient coefficients are zero (the value coefficients are 1 and 0)"""
    return np.zeros((nB, nc)), np.zeros((nB, nc))
