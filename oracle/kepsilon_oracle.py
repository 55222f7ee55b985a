"""CPU restatement (numpy over the oracle's primitives) of the standard k-epsilon model's transport step -- TEST INFRASTRUCTURE
(the checker of rapidcfd-dev_b200/kepsilon.py; never imported by the product).

  kEpsilon::correct      src/turbulenceModels/incompressible/RAS/kEpsilon/kEpsilon.C:227-276
  DkEff / DepsilonEff    kEpsilon.H:123-138   (nut + nu, nut/sigmaEps + nu)
  bound                  FV/cfdTools/general/bound/bound.C:33-72
  fvc::average           FV/finiteVolume/fvc/fvcAverage.C:43-114 (surfaceSum(magSf*ssf)/surfaceSum(magSf) of the linear face values)
  fvm::Sp, operator==, operator-(field, matrix)   FV/finiteVolume/fvm/fvmSup.C:100-150, fvMatrix.C:1750-2350
  symm, magSqr           OpenFOAM/primitives/Tensor/TensorI.H:483-491, SymmTensor/SymmTensorI.H:276-284
Scope: the two transport solves and nut on a single domain with fixedValue boundary values of k and epsilon on every patch -- no
wall functions (epsilon_.boundaryField().updateCoeffs() / boundaryManipulate are those and are not restated).  The statement
order follows kEpsilon.C; the file itself cannot be compiled here (it needs the RASModel class tree), so this composition is
UNPINNED; the operators it is made of are pinned one by one (DESIGN.md section 2)."""
import numpy as np

from oracle import fvm_oracle as fo

SMALL = 1e-15


def symm_magsqr(T):
    """magSqr(symm(T)), T [n, 9] row-major"""
    T = np.asarray(T, float).reshape(-1, 9)
    xx, yy, zz = T[:, 0], T[:, 4], T[:, 8]
    xy, xz, yz = 0.5 * (T[:, 1] + T[:, 3]), 0.5 * (T[:, 2] + T[:, 6]), 0.5 * (T[:, 5] + T[:, 7])
    s = xx * xx
    s = s + 2.0 * (xy * xy)
    s = s + 2.0 * (xz * xz)
    s = s + yy * yy
    s = s + 2.0 * (yz * yz)
    return s + zz * zz


class KEpsilon:
    def __init__(self, orc, addr, Sf, magSf, w, delta, V, bfc, bSf, bMagSf, bDelta, Ub, nu, k, epsilon, kB, epsB, Cmu=0.09, C1=1.44,
                 C2=1.92, sigmaEps=1.3, kMin=SMALL, epsilonMin=SMALL):
        self.orc, self.addr = orc, addr
        f = lambda x: np.array(x, float)
        self.Sf, self.magSf, self.w, self.delta, self.V = f(Sf), f(magSf), f(w), f(delta), f(V)
        self.bfc, self.bSf, self.bMagSf, self.bDelta, self.Ub = np.asarray(bfc, np.int32), f(bSf), f(bMagSf), f(bDelta), f(Ub)
        self.nu, self.Cmu, self.C1, self.C2, self.sigmaEps, self.kMin, self.epsilonMin = nu, Cmu, C1, C2, sigmaEps, kMin, epsilonMin
        self.k, self.epsilon, self.kB, self.epsB = f(k), f(epsilon), f(kB), f(epsB)
        # constructor body (kEpsilon.C:134-141): bound both, then nut
        self.bound("k", kMin)
        self.bound("epsilon", epsilonMin)
        self.update_nut()

    def update_nut(self):
        self.nut = (self.Cmu * (self.k * self.k)) / self.epsilon
        self.nutB = (self.Cmu * (self.kB * self.kB)) / self.epsB

    def bound(self, which, lowerBound):
        vsf, vb = getattr(self, which), getattr(self, which + "B" if which == "k" else "epsB")
        mx, mxb = fo.max_(vsf, lowerBound), fo.max_(vb, lowerBound)
        face = np.asarray(self.orc.interpolate_linear(self.addr, self.w, mx, 1))
        num = np.asarray(self.orc.surface_integrate(self.addr, self.magSf * face, self.bfc, self.bMagSf * mxb, self.V, 1, False, 1))
        den = np.asarray(self.orc.surface_integrate(self.addr, self.magSf, self.bfc, self.bMagSf, self.V, 1, False, 1))
        av = num / den
        new = fo.max_(fo.max_(vsf, av * np.where(-vsf >= 0, 1.0, 0.0)), lowerBound)
        setattr(self, which, new)
        setattr(self, "kB" if which == "k" else "epsB", mxb)

    def _transport(self, psi, psiB, gamma, gammaB, su, sp, phi, bphi, rDeltaT, divScheme, alpha, ctl):
        orc = self.orc
        ddtDiag, ddtSource = rDeltaT * self.V, (rDeltaT * psi) * self.V
        wConv = np.where(phi >= 0, 1.0, 0.0) if divScheme == "upwind" else self.w
        cLower, cUpper, cDiag = (np.asarray(x) for x in orc.convection_fill(self.addr, wConv, phi))
        gf = np.asarray(orc.interpolate_linear(self.addr, self.w, gamma, 1))
        lUpper, lDiag = (np.asarray(x) for x in orc.laplacian_fill(self.addr, self.delta, gf * self.magSf))
        diag, upper, lower = (ddtDiag + cDiag) - lDiag, cUpper - lUpper, cLower - lUpper
        lIc, lBc = fo.fixedValue_laplacian_coeffs(gammaB * self.bMagSf, self.bDelta, psiB[:, None])
        ic, bc = np.zeros_like(lIc) - lIc, ((-bphi) * psiB)[:, None] - lBc
        diag = diag + self.V * sp                     # == (su - fvm::Sp(sp, psi)): diag - (-(V*sp))
        source = ddtSource + self.V * su              #                            source - (-(V*su))
        eqn = fo.FvMatrix(orc, self.addr, 1, diag, upper, lower, source, psi, self.V, self.bfc, ic, bc)
        if alpha is not None:
            eqn.relax(alpha)
        out, perfs, _ = eqn.solve("PBiCG", "DILU", **ctl)
        return np.asarray(out).reshape(-1), perfs[0]

    def correct(self, U, phi, bphi, deltaT, divScheme="upwind", alphaEps=None, alphaK=None, controls=None):
        """kEpsilon::correct(): returns (perf of the epsilon solve, perf of the k solve)"""
        ctl = controls or dict(tolerance=1e-10, relTol=0.0)
        gradU = np.asarray(self.orc.gauss_grad(self.addr, self.Sf.ravel(), np.asarray(self.orc.interpolate_linear(
            self.addr, self.w, np.asarray(U, float).ravel(), 3)).ravel(), self.bfc, self.bSf.ravel(), self.Ub.ravel(), self.V, 3)).reshape(-1, 9)
        G = (self.nut * 2.0) * symm_magsqr(gradU)
        rDeltaT = 1.0 / deltaT
        self.epsilon, pe = self._transport(self.epsilon, self.epsB, self.nut / self.sigmaEps + self.nu, self.nutB / self.sigmaEps + self.nu,
                                           ((self.C1 * G) * self.epsilon) / self.k, (self.C2 * self.epsilon) / self.k, phi, bphi, rDeltaT,
                                           divScheme, alphaEps, ctl)
        self.bound("epsilon", self.epsilonMin)
        self.k, pk = self._transport(self.k, self.kB, self.nut + self.nu, self.nutB + self.nu, G, self.epsilon / self.k, phi, bphi, rDeltaT,
                                     divScheme, alphaK, ctl)
        self.bound("k", self.kMin)
        self.update_nut()
        self.G = G
        return pe, pk
