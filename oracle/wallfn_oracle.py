"""CPU restatement of the k-epsilon wall functions and of fvMatrix::setValues -- TEST INFRASTRUCTURE (the checker of
rapidcfd-dev_b200/kepsilon.py's wall-function path and of csrc/wallfn.cu; never imported by the product).

Paths: FV/ = src/finiteVolume/, WF/ = src/TurbulenceModels/turbulenceModels/RAS/derivedFvPatchFields/wallFunctions/.

  fvMatrix::setValues       FV/fvMatrices/fvMatrix/fvMatrix.C:940-950 -> setValuesFromList :456-657, functors :350-450.
                            PINNED: `ref_set_values` runs the reference's own code (oracle/_ref/libref_setvalues.so, built by
                            oracle/setvalues.mk from ref_harness/harness_setvalues.cpp) and tests/test_wall_functions_cpu.py
                            compares `set_values` with it bit for bit.
  nutkWallFunction          WF/nutWallFunctions/nutkWallFunction/nutkWallFunctionFvPatchScalarField.C:60-130 (calcNut),
                            yPlusLam WF/nutWallFunctions/nutWallFunction/nutWallFunctionFvPatchScalarField.C:154-168
  epsilonWallFunction       WF/epsilonWallFunctions/epsilonWallFunction/epsilonWallFunctionFvPatchScalarField.C:
                            createAveragingWeights :140-215, calculateTurbulenceFields :231-262, calculate :334-400,
                            updateCoeffs :540-590, manipulateMatrix :739-752 (setValues(faceCells, patchInternalField()))
  kqRWallFunction           WF/kqRWallFunctions/kqRWallFunction/kqRWallFunctionFvPatchField.C (zeroGradient)
  kEpsilon::correct         src/turbulenceModels/incompressible/RAS/kEpsilon/kEpsilon.C:227-276
The wall-function classes need the turbulence-model class tree and are restated, not compiled: that composition is UNPINNED
(DESIGN.md section 2).  Transcendental functions go through Python's math module (the C library's log / pow / sqrt), one value
at a time, so the host build of csrc/wallfn_kernels.cuh can be held to this file bit for bit.

Finding while restating setValues (mirrored, not corrected; reproduced by running the reference's code):
 * setValuesFromList asks the matrix for its non-const lower() (:574), which turns a symmetric matrix asymmetric with a copy of
   upper (lduMatrix.C:221-238); the `if (asymmetric())` of :612 then clears that copy too.  The result of a symmetric matrix is
   an asymmetric one: upper cleared where the owner is set, lower where the neighbour is set.
 * An unset cell subtracts lower[f]*value[nei] on its owner faces and upper[f]*value[own] on its neighbour faces: the
   coefficient of the OTHER row (stock OpenFOAM subtracts the cell's own row coefficient), and keeps its coupling to the set
   cell in the matrix (stock OpenFOAM clears it).  On a symmetric matrix the two readings agree on the source.
"""
import ctypes as C
import math
import os

import numpy as np

from oracle import fvm_oracle as fo
from oracle import kepsilon_oracle as ko

CMU, KAPPA, E = 0.09, 0.41, 9.8     # nutWallFunctionFvPatchScalarField.H / epsilonWallFunctionFvPatchScalarField.H defaults

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_SV = os.path.join(_HERE, "_ref", "libref_setvalues.so")
_libsv = None


# ---- fvMatrix::setValues ------------------------------------------------------------------------------------------------------
def set_values(om, cells, values):
    """setValuesFromList on an fvm_oracle.FvMatrix (scalar, single domain) in place: psi, source, upper, lower, ic, bc.
    A cell listed twice must carry equal values (the reference scatters them in no defined order)."""
    assert om.nc == 1 and not len(om.cfc), "setValues: scalar matrices on a single domain"
    cells, values = np.asarray(cells, np.int64), np.asarray(values, float)
    n = om.n
    om.psi[cells, 0] = values                                   # :471-480
    om.source[cells, 0] = values * om.diag[cells]               # :482-497
    if om.lower is None:                                        # lower() (:574) makes a symmetric matrix asymmetric
        om.lower = om.upper.copy()
    mask = np.zeros(n, bool)
    mask[cells] = True
    val = np.zeros(n)
    val[cells] = values
    l, u = np.asarray(om.addr.lower(), np.int64), np.asarray(om.addr.upper(), np.int64)
    ownMask, neiMask = mask[l], mask[u]
    # fvMatrixSetValuesSourceFunctor: per unset cell its owner faces (ascending), then its neighbour faces in losort order
    # (ascending face: losort is a stable sort by neighbour); np.subtract.at subtracts in that order, products rounded first
    s = om.source[:, 0].copy()
    f1 = np.nonzero(neiMask & ~mask[l])[0]
    np.subtract.at(s, l[f1], om.lower[f1] * val[u[f1]])
    f2 = np.nonzero(ownMask & ~mask[u])[0]
    np.subtract.at(s, u[f2], om.upper[f2] * val[l[f2]])
    om.source[:, 0] = s
    om.upper[ownMask] = 0.0                                     # :600-610
    om.lower[neiMask] = 0.0                                     # :612-622 (asymmetric by now)
    b = mask[om.bfc]                                            # :624-655
    om.ic[b] = 0.0
    om.bc[b] = 0.0


def ref_set_values(nCells, lower, upper, patchFaceCells, psi, diag, upperC, lowerC, source, ic, bc, calls):
    """The reference's setValues, called once per (cells, values) of `calls` on one fvMatrix<scalar>.  patchFaceCells: faceCells
    per patch; ic / bc flat over the patches.  Returns dict(psi, diag, upper, lower, source, ic, bc, asymmetric)."""
    from oracle import ref_ldu as rl
    global _libsv
    if _libsv is None:
        if not rl.available() or not os.path.exists(_LIB_SV):
            raise RuntimeError("oracle/_ref/libref_setvalues.so is not built (needs the reference tree)")
        _libsv = C.CDLL(_LIB_SV)
    l, u = rl._i(lower), rl._i(upper)
    n, nF = int(nCells), len(l)
    os_, ls, lo = (rl._i(x) for x in rl.ldu_arrays(n, l, u))
    ps = rl._i(np.concatenate([[0], np.cumsum([len(f) for f in patchFaceCells])]))
    fc = rl._i(np.concatenate([np.asarray(f, np.int32) for f in patchFaceCells]) if patchFaceCells else np.zeros(0, np.int32))
    cs = rl._i(np.concatenate([[0], np.cumsum([len(c) for c, _ in calls])]))
    cells = rl._i(np.concatenate([np.asarray(c, np.int32) for c, _ in calls]))
    vals = rl._d(np.concatenate([np.asarray(v, float) for _, v in calls]))
    psi, upperC, source, ic, bc = (rl._d(np.array(x, float)) for x in (psi, upperC, source, ic, bc))
    lowp = None if lowerC is None else rl._p(rl._d(np.array(lowerC, float)))
    diagOut, lowerOut = np.zeros(n), np.zeros(nF)
    rc = _libsv.ref_fvm_set_values(n, nF, rl._p(l), rl._p(u), rl._p(os_), rl._p(ls), rl._p(lo), len(patchFaceCells), rl._p(ps),
                                   rl._p(fc), rl._p(psi), rl._p(rl._d(diag)), rl._p(upperC), lowp, rl._p(source), rl._p(ic), rl._p(bc),
                                   len(calls), rl._p(cs), rl._p(cells), rl._p(vals), rl._p(diagOut), rl._p(lowerOut))
    if rc < 0:
        raise RuntimeError(f"ref_fvm_set_values failed ({rc})")
    return dict(psi=psi, diag=diagOut, upper=upperC, lower=lowerOut, source=source, ic=ic, bc=bc, asymmetric=rc == 2)


# ---- wall functions -----------------------------------------------------------------------------------------------------------
def _max(a, b):
    return a if a > b else b


def y_plus_lam(kappa=KAPPA, E=E):
    """nutWallFunctionFvPatchScalarField::yPlusLam: ypl = 11, then ten times log(max(E*ypl, 1))/kappa"""
    ypl = 11.0
    for _ in range(10):
        ypl = math.log(_max(E * ypl, 1.0)) / kappa
    return ypl


def constants(Cmu=CMU):
    """(Cmu25, Cmu75): pow025(Cmu) = sqrt(sqrt(Cmu)) (doubleScalar.H), pow(Cmu, 0.75)"""
    return math.sqrt(math.sqrt(Cmu)), math.pow(Cmu, 0.75)


def nutk(y, kc, nuw, yPlusLam, Cmu25, kappa=KAPPA, E=E):
    """nutkWallFunctionFvPatchScalarFieldFunctor per wall face: y, k of its cell, nu"""
    out = np.zeros(len(y))
    for i, (yi, ki) in enumerate(zip(np.asarray(y, float), np.asarray(kc, float))):
        yPlus = ((Cmu25 * yi) * math.sqrt(ki)) / nuw
        out[i] = nuw * (((yPlus * kappa) / math.log(E * yPlus)) - 1.0) if yPlus > yPlusLam else 0.0
    return out


def corner_weights(nCells, bfc, epsWall):
    """createAveragingWeights: per epsilon-wall face 1/(the number of epsilon-wall faces of its cell over all such patches);
    0 on every other boundary face (which the kernels read as `not an epsilon wall`)"""
    bfc, epsWall = np.asarray(bfc, np.int64), np.asarray(epsWall, bool)
    count = np.zeros(nCells)
    np.add.at(count, bfc[epsWall], 1.0)
    w = np.zeros(len(bfc))
    w[epsWall] = 1.0 / count[bfc[epsWall]]
    return w


def mag_sngrad(U, Ub, bfc, bDelta):
    """mag(Uw.snGrad()) of a fixedValue U patch: |deltaCoeffs*(Uw - U[faceCells])|, magSqr summed x, y, z"""
    g = np.asarray(bDelta, float)[:, None] * (np.asarray(Ub, float).reshape(-1, 3) - np.asarray(U, float).reshape(-1, 3)[bfc])
    return np.sqrt((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2])


def epsilon_wall(bfc, cw, y, k, U, Ub, bDelta, nutB, nu, G, epsilon, epsB, Cmu25, Cmu75, kappa=KAPPA):
    """epsilonWallFunction::updateCoeffs of all epsilon-wall patches: epsilon0 and G0 summed per cell over its wall faces (patch
    order, faces ascending: matrixPatchOperation), then G = G0 and epsilon = epsilon0 in the wall cells and the patch values
    epsilon0[faceCells].  Returns new (G, epsilon, epsB)."""
    bfc = np.asarray(bfc, np.int64)
    G, epsilon, epsB = (np.array(x, float) for x in (G, epsilon, epsB))
    mg = mag_sngrad(U, Ub, bfc, bDelta)
    eps0, G0, wall = {}, {}, np.asarray(cw) > 0
    for f in np.nonzero(wall)[0]:
        c = int(bfc[f])
        kc, d = float(k[c]), kappa * float(y[f])
        eps0[c] = eps0.get(c, 0.0) + ((cw[f] * Cmu75) * math.pow(kc, 1.5)) / d
        G0[c] = G0.get(c, 0.0) + ((((cw[f] * (float(nutB[f]) + nu)) * mg[f]) * Cmu25) * math.sqrt(kc)) / d
    for c in eps0:
        G[c], epsilon[c] = G0[c], eps0[c]
    epsB[wall] = epsilon[bfc[wall]]
    return G, epsilon, epsB


# ---- the k-epsilon step with wall functions -----------------------------------------------------------------------------------
class KEpsilonWall(ko.KEpsilon):
    """kepsilon_oracle.KEpsilon with per-patch boundary types of k / epsilon / nut (fixedValue, kqRWallFunction, epsilonWallFunction,
    nutkWallFunction) and the near-wall distance y
    per boundary face.  patchStart: offsets of the patches in the flat boundary list."""

    def __init__(self, orc, addr, Sf, magSf, w, delta, V, bfc, bSf, bMagSf, bDelta, Ub, nu, k, epsilon, kB, epsB, patchStart, kTypes,
                 epsTypes, nutTypes, y, **kw):
        self.ps = np.asarray(patchStart, np.int64)
        face = lambda types, t: np.repeat([x == t for x in types], np.diff(self.ps))
        self.zg = face(kTypes, "kqRWallFunction").astype(float)
        self.epsWall = face(epsTypes, "epsilonWallFunction")
        self.nutkFaces = np.nonzero(face(nutTypes, "nutkWallFunction"))[0]
        self.epsPatches = [p for p, t in enumerate(epsTypes) if t == "epsilonWallFunction"]
        self.y = np.asarray(y, float)
        self.Cmu25, self.Cmu75 = constants(kw.get("Cmu", CMU))
        self.yPlusLam = y_plus_lam()
        self.cw = corner_weights(len(V), bfc, self.epsWall)
        self.nCorrect = 0
        super().__init__(orc, addr, Sf, magSf, w, delta, V, bfc, bSf, bMagSf, bDelta, Ub, nu, k, epsilon, kB, epsB, **kw)

    def update_nut(self):
        super().update_nut()
        f = self.nutkFaces                  # nut.correctBoundaryConditions(): the nutk patches from k
        self.nutB[f] = nutk(self.y[f], self.k[self.bfc[f]], self.nu, self.yPlusLam, self.Cmu25)

    def _transport_wall(self, psi, old, psiB, gamma, gammaB, su, sp, phi, bphi, rDeltaT, divScheme, alpha, ctl, zg, setv):
        orc = self.orc
        ddtDiag, ddtSource = rDeltaT * self.V, (rDeltaT * old) * self.V
        wConv = np.where(phi >= 0, 1.0, 0.0) if divScheme == "upwind" else self.w
        cLower, cUpper, cDiag = (np.asarray(x) for x in orc.convection_fill(self.addr, wConv, phi))
        gf = np.asarray(orc.interpolate_linear(self.addr, self.w, gamma, 1))
        lUpper, lDiag = (np.asarray(x) for x in orc.laplacian_fill(self.addr, self.delta, gf * self.magSf))
        diag, upper, lower = (ddtDiag + cDiag) - lDiag, cUpper - lUpper, cLower - lUpper
        lIc, lBc = fo.fixedValue_laplacian_coeffs(gammaB * self.bMagSf, self.bDelta, psiB[:, None])
        ic, bc = np.zeros_like(lIc) - lIc, ((-bphi) * psiB)[:, None] - lBc
        if zg.any():                        # zeroGradient faces: laplacian coefficients 0, convection valueInternalCoeffs 1
            fv = 1.0 - zg
            ic, bc = (fv * ic[:, 0] + zg * bphi)[:, None], (fv * bc[:, 0])[:, None]
        diag = diag + self.V * sp
        source = ddtSource + self.V * su
        eqn = fo.FvMatrix(orc, self.addr, 1, diag, upper, lower, source, psi, self.V, self.bfc, ic, bc)
        if alpha is not None:
            eqn.relax(alpha)
        for p in setv:                      # boundaryManipulate: manipulateMatrix of each epsilon-wall patch in patch order
            cells = self.bfc[self.ps[p]:self.ps[p + 1]]
            set_values(eqn, cells, eqn.psi[cells, 0].copy())
        out, perfs, _ = eqn.solve("PBiCG", "DILU", **ctl)
        return np.asarray(out).reshape(-1), perfs[0]

    def correct(self, U, phi, bphi, deltaT, divScheme="upwind", alphaEps=None, alphaK=None, controls=None):
        ctl = controls or dict(tolerance=1e-10, relTol=0.0)
        gradU = np.asarray(self.orc.gauss_grad(self.addr, self.Sf.ravel(), np.asarray(self.orc.interpolate_linear(
            self.addr, self.w, np.asarray(U, float).ravel(), 3)).ravel(), self.bfc, self.bSf.ravel(), self.Ub.ravel(), self.V, 3)).reshape(-1, 9)
        G = (self.nut * 2.0) * ko.symm_magsqr(gradU)
        epsPre = self.epsilon
        if self.epsWall.any():              # epsilon_.boundaryField().updateCoeffs()
            G, self.epsilon, self.epsB = epsilon_wall(self.bfc, self.cw, self.y, self.k, U, self.Ub, self.bDelta, self.nutB, self.nu, G,
                                                      self.epsilon, self.epsB, self.Cmu25, self.Cmu75)
        # fvm::ddt's old value: boundaryField() stores the old time before updateCoeffs writes the wall cells -- once an old
        # field exists; the first oldTime() of a run copies the field as it is then (DESIGN.md section 8, f4)
        old = epsPre if self.nCorrect else self.epsilon
        rDeltaT = 1.0 / deltaT
        self.epsilon, pe = self._transport_wall(self.epsilon, old, self.epsB, self.nut / self.sigmaEps + self.nu,
                                                self.nutB / self.sigmaEps + self.nu, ((self.C1 * G) * self.epsilon) / self.k,
                                                (self.C2 * self.epsilon) / self.k, phi, bphi, rDeltaT, divScheme, alphaEps, ctl,
                                                np.zeros(len(self.bfc)), self.epsPatches)
        self.bound("epsilon", self.epsilonMin)
        self.k, pk = self._transport_wall(self.k, self.k, self.kB, self.nut + self.nu, self.nutB + self.nu, G, self.epsilon / self.k, phi,
                                          bphi, rDeltaT, divScheme, alphaK, ctl, self.zg, [])
        if self.zg.any():                   # the solve's correctBoundaryConditions: zeroGradient k takes its cell value
            self.kB = (1.0 - self.zg) * self.kB + self.zg * self.k[self.bfc]
        self.bound("k", self.kMin)
        self.update_nut()
        self.G = G
        self.nCorrect += 1
        return pe, pk
