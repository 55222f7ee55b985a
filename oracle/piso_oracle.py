"""CPU restatement of one icoFoam time step (SURVEY.md section 8(f) rank 2) -- TEST INFRASTRUCTURE ONLY.

Follows /root/reference/applications/solvers/incompressible/icoFoam/icoFoam.C:55-103 statement by statement, each
field expression evaluated as the reference's gpuField operators evaluate it: one rounded elementwise operation per
operator, in the written order (numpy does the same).  Schemes: ddt Euler, div Gauss linear, laplacian Gauss linear
uncorrected (orthogonal meshes), grad Gauss linear, interpolate linear -- the cavity tutorial's fvSchemes.  Boundary
conditions: U fixedValue on every boundary face, p zeroGradient (the lid-driven cavity); single domain.  The
pieces are pinned (matrix glue, coefficient fills, face sums, solvers, the Euler ddt statements:
tests/test_reference_functors.py); the step AS A WHOLE is PARITY UNPINNED (the application needs the whole library)
and is checked by the physics it has to produce (tests/test_oracle_piso.py).  FV/ = src/finiteVolume/.
"""
import numpy as np

from . import fvm_oracle as fo

SMALL = 1e-15   # src/OpenFOAM/primitives/Scalar/doubleScalar/doubleScalar.H


class Cavity:
    """mesh + fields of the case on one rank; arrays in OpenFOAM order (faces: owner-sorted upper triangle; boundary
    faces: the fixedValue patches concatenated in patch order, then -- on a decomposed case -- the processor patches
    in patch order: `cou*` arrays, flat over their faces)."""

    def __init__(self, orc, nCells, lower, upper, Sf, magSf, weights, deltaCoeffs, V, bFaceCells, bSf, bMagSf,
                 bDeltaCoeffs, Ub, nu, deltaT, pRefCell=0, pRefValue=0.0, couPatchStart=None, couFaceCells=None,
                 neighbRank=None, couSf=None, couMagSf=None, couWeights=None, couDeltaCoeffs=None, comm=None):
        self.orc, self.comm = orc, comm
        self.cfc = np.zeros(0, np.int64) if couFaceCells is None else np.asarray(couFaceCells, np.int64)
        if len(self.cfc):
            self.addr = orc.Addr(nCells, lower, upper, couPatchStart, couFaceCells, neighbRank=neighbRank)
        else:
            self.addr = orc.Addr(nCells, lower, upper)
        self.n, self.lower, self.upper = int(nCells), np.asarray(lower), np.asarray(upper)
        self.Sf, self.magSf, self.w, self.delta, self.V = (np.asarray(x, float) for x in (Sf, magSf, weights, deltaCoeffs, V))
        self.bfc = np.asarray(bFaceCells, np.int64)
        self.bSf, self.bMagSf, self.bDelta, self.Ub = (np.asarray(x, float) for x in (bSf, bMagSf, bDeltaCoeffs, Ub))
        nC = len(self.cfc)
        z = np.zeros(nC)
        self.cSf = np.zeros((nC, 3)) if couSf is None else np.asarray(couSf, float)
        self.cMagSf, self.cw, self.cDelta = (z if x is None else np.asarray(x, float) for x in (couMagSf, couWeights, couDeltaCoeffs))
        # every boundary face of the rank, as the face-sum functions take them
        self.allfc = np.concatenate([self.bfc, self.cfc]).astype(np.int32)
        self.allSf = np.concatenate([self.bSf, self.cSf])
        self.nu, self.deltaT, self.pRefCell, self.pRefValue = float(nu), float(deltaT), int(pRefCell), float(pRefValue)
        self.U = np.zeros((self.n, 3))
        self.p = np.zeros(self.n)
        # createPhi.H: phi = linearInterpolate(U) & mesh.Sf()
        self.phi = self.flux_of(self.U)
        self.bphi = self._dot(self.Ub, self.bSf)
        self.cphi = self._dot(self.interpolate_coupled(self.U), self.cSf)

    # ---- field expressions ----------------------------------------------------------------------------
    @staticmethod
    def _dot(a, b):            # Vector & Vector: x*x + y*y + z*z, left to right (VectorI.H)
        return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]

    def interpolate(self, vf):
        """linear: w*(vf[own] - vf[nei]) + vf[nei] (surfaceInterpolationScheme.C:272-351, the form interpolate(vf) uses)"""
        w = self.w if vf.ndim == 1 else self.w[:, None]
        return w * (vf[self.lower] - vf[self.upper]) + vf[self.upper]

    def pnf(self, vf):
        """patchNeighbourField of the processor patches, (nCoupledFaces[, 3])"""
        if not len(self.cfc):
            return np.zeros((0,) + vf.shape[1:])
        if vf.ndim == 1:
            return self.addr.patch_neighbour_field(np.ascontiguousarray(vf), self.comm)
        return np.stack([self.addr.patch_neighbour_field(np.ascontiguousarray(vf[:, k]), self.comm) for k in range(3)], axis=1)

    def interpolate_coupled(self, vf, pnf=None):
        """coupled patch faces: w*patchInternalField + (1 - w)*patchNeighbourField (:357-370)"""
        pnf = self.pnf(vf) if pnf is None else pnf
        w = self.cw if vf.ndim == 1 else self.cw[:, None]
        return w * vf[self.cfc] + (1 - w) * pnf

    def flux_of(self, U):
        return self._dot(self.interpolate(U), self.Sf)

    def grad(self, p):
        """fvc::grad = gaussGrad(linear): gradf(interpolate(p)) (gaussGrad.C:143-271); zeroGradient walls, interpolated
        values on the processor faces; the boundary correction of correctBoundaryConditions only touches the patch
        values of the gradient, which nothing here reads"""
        pb = np.concatenate([p[self.bfc], self.interpolate_coupled(p)])
        g = self.orc.gauss_grad(self.addr, self.Sf.ravel(), self.interpolate(p), self.allfc, self.allSf.ravel(), pb, self.V, 1)
        return np.asarray(g).reshape(self.n, 3)

    def div(self, phi, bphi, cphi=None):
        """fvc::div(flux) = surfaceIntegrate (fvcDiv.C, fvcSurfaceIntegrate.C:138-203)"""
        cphi = self.cphi if cphi is None else cphi
        return np.asarray(self.orc.surface_integrate(self.addr, phi, self.allfc, np.concatenate([bphi, cphi]), self.V, 1))

    # ---- one time step: icoFoam.C:55-103 --------------------------------------------------------------
    def step(self, nCorr=2, nNonOrthCorr=0, UControls=None, pControls=None, momentumPredictor=True,
             USolver=("PBiCG", "DILU"), pSolver=("PCG", "DIC"), gamg=None, divScheme="linear"):
        """USolver / pSolver: (solver, preconditioner or smoother) as fvSolution names them; gamg: the cached
        agglomeration (orc.Gamg) when pSolver is GAMG; divScheme "linear" | "upwind": the weights of fvm::div(phi, U)
        (upwind.H:120-123 pos(faceFlux), on the coupled patches too)"""
        orc = self.orc
        fvm = lambda nc, diag, upper, lower, source, psi, ic, bc, ci, cb: fo.FvMatrix(
            orc, self.addr, nc, diag, upper, lower, source, psi, self.V, self.bfc, ic, bc,
            couInt=ci if len(self.cfc) else None, couBou=cb if len(self.cfc) else None, comm=self.comm)
        U0, phi0, cphi0 = self.U.copy(), self.phi.copy(), self.cphi.copy()      # oldTime fields
        rDeltaT = 1.0 / self.deltaT
        # fvm::ddt(U): EulerDdtScheme.C:331-361
        ddtDiag = rDeltaT * self.V
        ddtSource = (rDeltaT * U0) * self.V[:, None]
        # fvm::div(phi, U): gaussConvectionScheme.C:76-115 (lower = -w*phi, upper = lower + phi, negSumDiag; fixedValue
        # patches: internalCoeffs = 0, boundaryCoeffs = -patchFlux*U_b; coupled: patchFlux*w and -patchFlux*(1 - w),
        # coupledFvPatchField.C:162-179)
        wConv = np.where(self.phi >= 0, 1.0, 0.0) if divScheme == "upwind" else self.w
        cwConv = np.where(self.cphi >= 0, 1.0, 0.0) if divScheme == "upwind" else self.cw
        cLower, cUpper, cDiag = orc.convection_fill(self.addr, wConv, self.phi)
        cIc = self.bphi[:, None] * np.zeros((len(self.bfc), 3))
        cBc = (-self.bphi)[:, None] * self.Ub
        cCi = self.cphi * cwConv
        cCb = (-self.cphi) * (1.0 - cwConv)
        # fvm::laplacian(nu, U): gaussLaplacianSchemes.C:39-93, gaussLaplacianScheme.C:46-89 (coupled: pGamma*(-delta) and
        # -pGamma*delta, coupledFvPatchField.C:184-209)
        gammaMagSf = self.nu * self.magSf
        lUpper, lDiag = orc.laplacian_fill(self.addr, self.delta, gammaMagSf)
        lIc, lBc = fo.fixedValue_laplacian_coeffs(self.nu * self.bMagSf, self.bDelta, self.Ub)
        cGamma = self.nu * self.cMagSf
        lCi = cGamma * (-self.cDelta)
        lCb = (-cGamma) * self.cDelta
        # UEqn = ddt + div - laplacian (fvMatrix.C operator+ / operator-: coefficient arrays added then subtracted)
        diag = (ddtDiag + cDiag) - lDiag
        upper = cUpper - lUpper
        lower = cLower - lUpper
        source = ddtSource
        ic, bc = cIc - lIc, cBc - lBc
        ci, cb = cCi - lCi, cCb - lCb
        perfs = {}
        if momentumPredictor:
            # solve(UEqn == -fvc::grad(p)): source += V*(-grad p) (fvMatrix.C operator==, operator-)
            src = source + self.V[:, None] * (-self.grad(self.p))
            UEqn = fvm(3, diag, upper, lower, src, self.U, ic, bc, ci, cb)
            self.U, perfs["U"], _ = UEqn.solve(USolver[0], USolver[1], **(UControls or dict(tolerance=1e-5, relTol=0.0)))
        cont = []
        for corr in range(nCorr):
            UEqn = fvm(3, diag, upper, lower, source, self.U, ic, bc, ci, cb)
            rAU = 1.0 / UEqn.A()
            HbyA = rAU[:, None] * UEqn.H()
            # phiHbyA = (interpolate(HbyA) & Sf) + interpolate(rAU)*ddtCorr(U, phi)
            phiCorr = phi0 - self._dot(self.Sf, self.interpolate(U0))             # EulerDdtScheme.C:536-539
            coeff = 1.0 - fo.min_(np.abs(phiCorr) / (np.abs(phi0) + SMALL), 1.0)      # ddtScheme.C:139-152
            ddtCorr = (coeff * rDeltaT) * phiCorr
            rAUf = self.interpolate(rAU)
            phiHbyA = self.flux_of(HbyA) + rAUf * ddtCorr
            bphiHbyA = self._dot(self.Ub, self.bSf)        # fixedValue: HbyA_b = U_b, coupling coefficient 0 (:156-162)
            # the same expression on the processor faces (their coupling coefficient is not zeroed)
            cphiCorr = cphi0 - self._dot(self.cSf, self.interpolate_coupled(U0))
            ccoeff = 1.0 - fo.min_(np.abs(cphiCorr) / (np.abs(cphi0) + SMALL), 1.0)
            crAUf = self.interpolate_coupled(rAU)
            cphiHbyA = self._dot(self.interpolate_coupled(HbyA), self.cSf) + crAUf * ((ccoeff * rDeltaT) * cphiCorr)
            # adjustPhi: closed domain, the boundary flux is U_b & Sf_b = 0: nothing to adjust (adjustPhi.C)
            for nonOrth in range(nNonOrthCorr + 1):
                # pEqn: fvm::laplacian(rAU, p) == fvc::div(phiHbyA)
                pUpper, pDiag = orc.laplacian_fill(self.addr, self.delta, rAUf * self.magSf)
                pGamma = crAUf * self.cMagSf
                pCi, pCb = pGamma * (-self.cDelta), (-pGamma) * self.cDelta
                pSource = np.zeros(self.n) + self.V * self.div(phiHbyA, bphiHbyA, cphiHbyA)
                zero = np.zeros((len(self.bfc), 1))
                pEqn = fvm(1, pDiag, pUpper, None, pSource, self.p, zero, zero, pCi, pCb)
                pEqn.setReference(self.pRefCell, self.pRefValue)
                psi, perf, _ = pEqn.solve(pSolver[0], pSolver[1], gamg, **(pControls or dict(tolerance=1e-6, relTol=0.0)))
                self.p = psi[:, 0]
                perfs.setdefault("p", []).append(perf[0])
                if nonOrth == nNonOrthCorr:
                    pEqn.psi = psi
                    internal, boundary, coupled = pEqn.flux()
                    self.phi = phiHbyA - internal[:, 0]
                    self.bphi = bphiHbyA - boundary[:, 0]
                    self.cphi = cphiHbyA - coupled[:, 0]
            # continuityErrs.H (global sums over the ranks)
            contErr = self.div(self.phi, self.bphi, self.cphi)
            tot = self._gsum3((np.abs(contErr) * self.V).sum(), (contErr * self.V).sum(), self.V.sum())
            cont.append((self.deltaT * tot[0] / tot[2], self.deltaT * tot[1] / tot[2]))
            # U = HbyA - rAU*fvc::grad(p); U.correctBoundaryConditions() (fixedValue: unchanged)
            self.U = HbyA - rAU[:, None] * self.grad(self.p)
        return perfs, cont

    # ---- one SIMPLE iteration: simpleFoam/UEqn.H:1-17, pEqn.H:1-40 (laminar, single domain) --------------
    def simple_step(self, alphaU=0.7, alphaP=0.3, divScheme="upwind", UControls=None, pControls=None,
                    USolver=("PBiCG", "DILU"), pSolver=("PCG", "DIC"), gamg=None, nNonOrthCorr=0):
        """UEqn = fvm::div(phi, U) - fvm::laplacian(nu, U) (the laminar divDevReff without its explicit transpose term);
        UEqn.relax(alphaU); solve(UEqn == -grad p); p from laplacian(rAU, p) == div(phiHbyA); phi = phiHbyA - pEqn.flux();
        p.relax(alphaP); U = HbyA - rAU*grad p.  divScheme: "upwind" (bounded Gauss upwind of the pitzDaily tutorial:
        weights pos(phi), upwind.H:120-123) or "linear"."""
        assert not len(self.cfc), "the SIMPLE restatement is single-domain"
        from . import limiters_oracle as lo
        orc = self.orc
        fvm = lambda nc, diag, upper, lower, source, psi, ic, bc: fo.FvMatrix(
            orc, self.addr, nc, diag, upper, lower, source, psi, self.V, self.bfc, ic, bc, couInt=None, couBou=None, comm=self.comm)
        wConv = lo.limited_weights(self.phi) if divScheme == "upwind" else self.w
        cLower, cUpper, cDiag = orc.convection_fill(self.addr, wConv, self.phi)
        cIc = self.bphi[:, None] * np.zeros((len(self.bfc), 3))
        cBc = (-self.bphi)[:, None] * self.Ub
        lUpper, lDiag = orc.laplacian_fill(self.addr, self.delta, self.nu * self.magSf)
        lIc, lBc = fo.fixedValue_laplacian_coeffs(self.nu * self.bMagSf, self.bDelta, self.Ub)
        diag = cDiag - lDiag
        upper = cUpper - lUpper
        lower = cLower - lUpper
        source = np.zeros((self.n, 3))
        ic, bc = cIc - lIc, cBc - lBc
        UEqn = fvm(3, diag, upper, lower, source, self.U, ic, bc)
        UEqn.relax(alphaU)                                    # fvMatrix.C:1088-1345: in place on diag and source
        diag, source = UEqn.diag, UEqn.source
        perfs = {}
        src = source + self.V[:, None] * (-self.grad(self.p))
        UEqnP = fvm(3, diag, upper, lower, src, self.U, ic, bc)
        self.U, perfs["U"], _ = UEqnP.solve(USolver[0], USolver[1], **(UControls or dict(tolerance=1e-5, relTol=0.1)))
        UEqn = fvm(3, diag, upper, lower, source, self.U, ic, bc)
        rAU = 1.0 / UEqn.A()
        HbyA = rAU[:, None] * UEqn.H()
        phiHbyA = self.flux_of(HbyA)
        bphiHbyA = self._dot(self.Ub, self.bSf)
        rAUf = self.interpolate(rAU)
        pOld = self.p.copy()                                  # p.storePrevIter() (simpleFoam.C)
        for nonOrth in range(nNonOrthCorr + 1):
            pUpper, pDiag = orc.laplacian_fill(self.addr, self.delta, rAUf * self.magSf)
            pSource = np.zeros(self.n) + self.V * self.div(phiHbyA, bphiHbyA)
            zero = np.zeros((len(self.bfc), 1))
            pEqn = fvm(1, pDiag, pUpper, None, pSource, self.p, zero, zero)
            pEqn.setReference(self.pRefCell, self.pRefValue)
            psi, perf, _ = pEqn.solve(pSolver[0], pSolver[1], gamg, **(pControls or dict(tolerance=1e-6, relTol=0.05)))
            self.p = psi[:, 0]
            perfs.setdefault("p", []).append(perf[0])
            if nonOrth == nNonOrthCorr:
                pEqn.psi = psi
                internal, boundary, _ = pEqn.flux()
                self.phi = phiHbyA - internal[:, 0]
                self.bphi = bphiHbyA - boundary[:, 0]
        contErr = self.div(self.phi, self.bphi)
        tot = self._gsum3((np.abs(contErr) * self.V).sum(), (contErr * self.V).sum(), self.V.sum())
        cont = (tot[0] / tot[2], tot[1] / tot[2])             # steady: deltaT = 1 (continuityErrs.H)
        self.p = pOld + alphaP * (self.p - pOld)              # GeometricField::relax: prevIter + alpha*(this - prevIter)
        self.U = HbyA - rAU[:, None] * self.grad(self.p)
        return perfs, cont

    def _gsum3(self, a, b, c):
        v = np.array([float(a), float(b), float(c)])
        if self.comm is None:
            return v
        out = v.copy()
        self.orc.lib().orc_comm_sum(self.comm.ptr(), self.orc._d(out), 3)
        return out


def cavity_from_hex(orc, meshmod, n, nu=0.01, deltaT=None, lid=(1.0, 0.0, 0.0)):
    """the lid-driven cavity on the synthetic n^3 hex mesh of rapidcfd-dev_b200/mesh.py (patch `movingWall` = +y)"""
    m = meshmod.hex_mesh(n)
    bfc = np.concatenate([p.faceCells for p in m.patches]).astype(np.int32)
    bSf = np.concatenate([p.Sf for p in m.patches])
    Ub = np.concatenate([np.tile(lid if p.name == "movingWall" else (0.0, 0.0, 0.0), (len(p.faceCells), 1))
                         for p in m.patches])
    nB = len(bfc)
    deltaT = deltaT if deltaT is not None else 0.5 * m.h / max(abs(v) for v in lid)     # Co = 0.5 at the lid
    return m, Cavity(orc, m.nCells, m.lower, m.upper, m.Sf(), m.magSf(), m.weights(), m.deltaCoeffs(), m.volumes(), bfc,
                     bSf, np.full(nB, m.h * m.h), np.full(nB, 2.0 / m.h), Ub, nu, deltaT)


def cavity_rank(orc, meshmod, n, nRanks, rank, comm, nu=0.01, deltaT=None, lid=(1.0, 0.0, 0.0)):
    """rank `rank` of the brick decomposition of the same cavity (mesh.decompose): fixedValue walls + processor patches;
    the pressure reference cell is global cell 0 (setRefCell: the rank that owns it, -1 elsewhere)"""
    m = meshmod.decompose(n, nRanks, rank)
    walls, procs = m.wall_patches(), m.coupled_patches()
    bfc = np.concatenate([p.faceCells for p in walls]).astype(np.int32)
    bSf = np.concatenate([p.Sf for p in walls])
    Ub = np.concatenate([np.tile(lid if p.name == "movingWall" else (0.0, 0.0, 0.0), (len(p.faceCells), 1)) for p in walls])
    nB = len(bfc)
    ps, fc = m.patch_start_facecells()
    nC = len(fc)
    deltaT = deltaT if deltaT is not None else 0.5 * m.h / max(abs(v) for v in lid)
    ref = np.nonzero(m.cellGlobal == 0)[0]
    return m, Cavity(orc, m.nCells, m.lower, m.upper, m.Sf(), m.magSf(), m.weights(), m.deltaCoeffs(), m.volumes(), bfc,
                     bSf, np.full(nB, m.h * m.h), np.full(nB, 2.0 / m.h), Ub, nu, deltaT,
                     pRefCell=int(ref[0]) if len(ref) else -1, couPatchStart=ps, couFaceCells=fc,
                     neighbRank=[p.neighbRank for p in procs], couSf=np.concatenate([p.Sf for p in procs]),
                     couMagSf=np.full(nC, m.h * m.h), couWeights=np.full(nC, 0.5), couDeltaCoeffs=np.full(nC, 1.0 / m.h),
                     comm=comm)
