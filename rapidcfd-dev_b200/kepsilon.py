"""The standard k-epsilon model's transport step sequenced over the C ABI (host side: sequencing only, every field stays on the
device): the production term, the two scalar transport equations -- each assembled from the coefficient-fill kernels and solved
by PBiCG + DILU through the fvMatrix glue, i.e. through the same boundary as every other solve -- the bounding of k and epsilon,
and nut.  `capi` is rapidcfd-dev_b200.capi (or the oracle-backed stand-in of tests/oracle_backend.py).

  kEpsilon::correct      src/turbulenceModels/incompressible/RAS/kEpsilon/kEpsilon.C:227-276
  DkEff / DepsilonEff    kEpsilon.H:123-138
  bound                  FV/cfdTools/general/bound/bound.C:33-72 (applied unconditionally: where no value lies below the bound the
                         expression returns the field unchanged, which is what the reference's `if (minVsf < lowerBound)` skips)
  wall functions         kqRWallFunction (zeroGradient k), epsilonWallFunction (updateCoeffs + manipulateMatrix -> fvMatrix::setValues,
                         csrc/wallfn.cu, csrc/fvmatrix.cu), nutkWallFunction (calcNut, csrc/wallfn.cu); WF/ lines in include/b200ldu.h
Scope: single domain; per patch fixedValue or a wall function for k, epsilon and nut (`kTypes`, `epsTypes`, `nutTypes`; without
them every patch is fixedValue, as before); div schemes upwind | linear."""
import math

import numpy as np

SMALL = 1e-15
KAPPA, E = 0.41, 9.8                  # the wall-function classes' defaults
PATCH_TYPES = dict(k=("fixedValue", "kqRWallFunction"), epsilon=("fixedValue", "epsilonWallFunction"),
                   nut=("fixedValue", "nutkWallFunction"))


def y_plus_lam(kappa=KAPPA, E=E):
    """nutWallFunctionFvPatchScalarField::yPlusLam (nutWallFunctionFvPatchScalarField.C:154-168), once per model"""
    ypl = 11.0
    for _ in range(10):
        ypl = math.log(max(E * ypl, 1.0)) / kappa
    return ypl


def corner_weights(nCells, bfc, epsWall):
    """createAveragingWeights (epsilonWallFunctionFvPatchScalarField.C:140-215): per epsilon-wall face 1/(the number of epsilon-wall
    faces of its cell over all such patches), 0 on the other boundary faces; once per mesh"""
    count = np.zeros(nCells)
    np.add.at(count, bfc[epsWall], 1.0)
    w = np.zeros(len(bfc))
    w[epsWall] = 1.0 / count[bfc[epsWall]]
    return w


class KEpsilon:
    def __init__(self, capi, case, bMagSf, bDeltaCoeffs, k, epsilon, kB, epsB, Cmu=0.09, C1=1.44, C2=1.92, sigmaEps=1.3, kMin=SMALL,
                 epsilonMin=SMALL, patchStart=None, kTypes=None, epsTypes=None, nutTypes=None, y=None):
        """case: the IcoFoam object that owns the mesh arrays on the device (addr, Sf, magSf, w, delta, V, bSf, Ub, nu).
        Wall functions: patchStart (offsets of the patches in the flat boundary list), the patch types of k, epsilon and nut
        (PATCH_TYPES; a missing list is fixedValue everywhere) and y, the near-wall distance of every boundary face
        (foamfile.PolyMesh.near_wall_dist)."""
        assert not case.nC, "k-epsilon step: single domain"
        self.capi, self.case, self.ops = capi, case, case.ops
        t = case._t
        self.bMagSf, self.bDelta = t(bMagSf), t(bDeltaCoeffs)
        self.k, self.epsilon, self.kB, self.epsB = t(k), t(epsilon), t(kB), t(epsB)
        self.Cmu, self.C1, self.C2, self.sigmaEps, self.kMin, self.epsilonMin = Cmu, C1, C2, sigmaEps, kMin, epsilonMin
        self._walls(patchStart, dict(k=kTypes, epsilon=epsTypes, nut=nutTypes), y)
        self.mat = capi.LduMatrix(case.addr)
        o = self.ops
        # surfaceSum(magSf): the denominator of fvc::average, constant
        self.sumMagSf = capi.fv_surface_integrate(case.addr, 1, case.magSf, self.bMagSf, case.V, False, 1)
        self.zeroB = o.smul(0.0, self.bMagSf)
        # constructor body (kEpsilon.C:134-141)
        self.k, self.kB = self.bound(self.k, self.kB, kMin)
        self.epsilon, self.epsB = self.bound(self.epsilon, self.epsB, epsilonMin)
        self.update_nut()

    def _walls(self, patchStart, types, y):
        """the per-mesh set-up of the wall functions: face masks, corner weights, yPlusLam, the cells of each epsilon-wall patch"""
        self.walls = any(v is not None for v in types.values())
        if not self.walls:
            return
        c, t = self.case, self.case._t
        ps = np.asarray(patchStart, np.int64)
        for field, names in types.items():
            for p, nm in enumerate(names or ()):
                if nm not in PATCH_TYPES[field]:
                    raise ValueError(f"Unknown patchField type {nm} for patch {p} of {field}\n\nValid patchField types are :\n"
                                     f"({' '.join(PATCH_TYPES[field])})")
            if names is not None and len(names) != len(ps) - 1:
                raise ValueError(f"{field}: {len(names)} patch types for {len(ps) - 1} patches")
        face = lambda field, nm: np.repeat([x == nm for x in (types[field] or ())], np.diff(ps)) if types[field] else \
            np.zeros(int(ps[-1]), bool)
        bfc = c.bfc.cpu().numpy().astype(np.int64)
        kq, epsWall, nutk = face("k", "kqRWallFunction"), face("epsilon", "epsilonWallFunction"), face("nut", "nutkWallFunction")
        i32 = lambda a: c.torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(c.ctx.device)
        self.zg = t(kq.astype(float)) if kq.any() else None
        self.cw = t(corner_weights(c.n, bfc, epsWall)) if epsWall.any() else None
        self.epsCells = [i32(bfc[ps[p]:ps[p + 1]]) for p, nm in enumerate(types["epsilon"] or ()) if nm == "epsilonWallFunction"]
        self.nutkFaces = i32(np.nonzero(nutk)[0]) if nutk.any() else None
        self.y = t(np.asarray(y, float)) if (epsWall.any() or nutk.any()) else None
        self.Cmu25, self.Cmu75 = math.sqrt(math.sqrt(self.Cmu)), math.pow(self.Cmu, 0.75)
        self.yPlusLam = y_plus_lam()
        self.nCorrect = 0

    def update_nut(self):
        o = self.ops
        self.nut = o.div(o.smul(self.Cmu, o.mul(self.k, self.k)), self.epsilon)
        self.nutB = o.div(o.smul(self.Cmu, o.mul(self.kB, self.kB)), self.epsB)
        if self.walls and self.nutkFaces is not None:       # nut.correctBoundaryConditions(): the nutk patches from k
            self.capi.wallfn_nutk(self.case.addr, self.nutkFaces, self.y, self.k, self.case.nu, self.yPlusLam, self.Cmu25, self.nutB)

    def bound(self, vsf, vb, lowerBound):
        capi, c, o = self.capi, self.case, self.ops
        mx, mxb = o.smax(vsf, lowerBound), o.smax(vb, lowerBound)
        face = capi.fv_interpolate_linear(c.addr, 1, c.w, mx)
        num = capi.fv_surface_integrate(c.addr, 1, o.mul(c.magSf, face), o.mul(self.bMagSf, mxb), c.V, False, 1)
        av = o.div(num, self.sumMagSf)
        return o.smax(o.bmax(vsf, o.mul(av, o.pos(o.neg(vsf)))), lowerBound), mxb

    def _transport(self, psi, psiB, gamma, gammaB, su, sp, phi, bphi, rDeltaT, divScheme, alpha, ctl, old=None, zg=None, setv=()):
        """old: the old-time value of fvm::ddt (psi when None); zg: 1 on zeroGradient (kqRWallFunction) faces; setv: the cells of
        each epsilon-wall patch, set to their values after relax (boundaryManipulate)"""
        capi, c, o = self.capi, self.case, self.ops
        a = c.addr
        ddtDiag, ddtSource = o.smul(rDeltaT, c.V), o.mul(o.smul(rDeltaT, psi if old is None else old), c.V)
        if divScheme not in ("upwind", "linear"):
            raise ValueError(f"Unknown discretisation scheme {divScheme}\n\nValid schemes are :\n(linear upwind)")
        wConv = capi.fv_limited_weights(c.ctx, phi) if divScheme == "upwind" else c.w
        cLower, cUpper, cDiag = capi.fv_convection_fill(a, wConv, phi)
        gf = capi.fv_interpolate_linear(a, 1, c.w, gamma)
        lUpper, lDiag = capi.fv_laplacian_fill(a, c.delta, o.mul(gf, c.magSf))
        diag, upper, lower = o.sub(o.add(ddtDiag, cDiag), lDiag), o.sub(cUpper, lUpper), o.sub(cLower, lUpper)
        gb = o.mul(gammaB, self.bMagSf)
        lIc, lBc = o.mul(gb, o.neg(self.bDelta)), o.mul(o.neg(gb), o.mul(self.bDelta, psiB))
        ic, bc = o.sub(self.zeroB, lIc), o.sub(o.mul(o.neg(bphi), psiB), lBc)
        if zg is not None:                       # zeroGradient: laplacian coefficients 0, convection valueInternalCoeffs 1
            fv = o.rsub(1.0, zg)
            ic, bc = o.add(o.mul(fv, ic), o.mul(zg, bphi)), o.mul(fv, bc)
        diag = o.add(diag, o.mul(c.V, sp))
        source = o.add(ddtSource, o.mul(c.V, su))
        self.mat.set(diag, upper, lower)
        new = psi.clone()
        eqn = capi.FvMatrix(self.mat, 1, diag, source, new, c.V, ic, bc)
        if alpha is not None:
            eqn.relax(alpha)                     # in place on diag / source (fvMatrix.C:1088-1345) ...
        for cells in setv:                       # manipulateMatrix of each epsilon-wall patch: setValues(faceCells, patchInternalField())
            eqn.setValues(cells, o.gather(cells, new), upper, lower)
        if alpha is not None or setv:
            self.mat.set(diag, upper, lower)     # ... and the matrix holds copies: it takes the changed coefficients here
        perf = eqn.solve("PBiCG", "DILU", **ctl)[0]
        return new, perf

    def correct(self, U, phi, bphi, deltaT, divScheme="upwind", alphaEps=None, alphaK=None, controls=None):
        """kEpsilon::correct(): returns (perf of the epsilon solve, perf of the k solve)"""
        capi, c, o = self.capi, self.case, self.ops
        ctl = controls or dict(tolerance=1e-10, relTol=0.0)
        gradU = capi.fv_grad_linear(c.addr, 3, c.Sf, c.w, U, c.bSf, c.Ub, c.V)
        self.G = G = o.mul(o.smul(2.0, self.nut), o.symm_magsqr(gradU))
        rDeltaT = 1.0 / deltaT
        nu = c.nu
        walls = dict(old=None, setv=())
        if self.walls:
            if self.cw is not None:              # epsilon_.boundaryField().updateCoeffs(): G and epsilon in the wall cells
                epsPre, self.epsilon, self.epsB = self.epsilon, self.epsilon.clone(), self.epsB.clone()
                capi.wallfn_epsilon(c.addr, self.cw, self.y, self.k, U, c.Ub, self.bDelta, self.nutB, nu, self.Cmu25, self.Cmu75, G,
                                    self.epsilon, self.epsB)
                # fvm::ddt's old value: boundaryField() stores the old time before updateCoeffs writes the wall cells
                # (GeometricField.C:740-767), once an old field exists; the first oldTime() copies the field as it is then (:810-834)
                walls = dict(old=epsPre if self.nCorrect else self.epsilon, setv=self.epsCells)
            self.nCorrect += 1
        self.epsilon, pe = self._transport(self.epsilon, self.epsB, o.sadd(o.sdiv(self.nut, self.sigmaEps), nu),
                                           o.sadd(o.sdiv(self.nutB, self.sigmaEps), nu),
                                           o.div(o.mul(o.smul(self.C1, G), self.epsilon), self.k),
                                           o.div(o.smul(self.C2, self.epsilon), self.k), phi, bphi, rDeltaT, divScheme, alphaEps, ctl,
                                           **walls)
        self.epsilon, self.epsB = self.bound(self.epsilon, self.epsB, self.epsilonMin)
        zg = self.zg if self.walls else None
        self.k, pk = self._transport(self.k, self.kB, o.sadd(self.nut, nu), o.sadd(self.nutB, nu), G, o.div(self.epsilon, self.k), phi,
                                     bphi, rDeltaT, divScheme, alphaK, ctl, zg=zg)
        if zg is not None:                       # the solve's correctBoundaryConditions: zeroGradient k takes its cell value
            self.kB = o.add(o.mul(o.rsub(1.0, zg), self.kB), o.mul(zg, o.gather(c.bfc, self.k)))
        self.k, self.kB = self.bound(self.k, self.kB, self.kMin)
        self.update_nut()
        return pe, pk

    def close(self):
        self.mat.close()
