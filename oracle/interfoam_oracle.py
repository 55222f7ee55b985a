"""CPU restatement (numpy over the oracle's primitives) of the interFoam phase-fraction step -- TEST INFRASTRUCTURE (the checker
of b200ldu_fv_limited_flux, b200ldu_vof_interface_flux and rapidcfd-dev_b200/interfoam.py; never imported by the product).

  alphaEqn.H, alphaEqnSubCycle.H      applications/solvers/multiphase/interFoam/
  interfaceProperties::calculateK     src/transportModels/interfaceProperties/interfaceProperties.C:118-159; deltaN :181-185
  fvc::flux(phi, vf, scheme)          gaussConvectionScheme.C:74-84 over limitedSurfaceInterpolationScheme.C:155-212
  boundary values of fvc::grad        gaussGrad.C:277-303
  Vector / (mag(Vector) + d), &       VectorSpaceI.H:336-355, :621-630, VectorI.H operator&
Every operator is one fp64 rounding in the reference's order.  The pieces this composes -- orc_interpolate_linear, orc_gauss_grad,
orc_surface_integrate, the limiter functions, mules_oracle, fvm_oracle, the Euler ddt and upwind convection fills -- are pinned one
by one; alphaEqn.H is an application fragment and interfaceProperties.C needs the GeometricField / fvc class tree, so this
COMPOSITION IS UNPINNED (DESIGN.md section 2).  Scope as the product step: static mesh, single domain, alpha1 zeroGradient."""
import numpy as np

from oracle import fvm_oracle as fo
from oracle import limiters_oracle as lo
from oracle import mules_oracle as mo


def limited_flux(scheme, lower, upper, faceFlux, vf, gradc, centres, cdWeights, k=1.0, fluxSign=1, outSign=1):
    """outSign*fvc::flux(fluxSign*faceFlux, vf, scheme) on the internal faces: the four-step composition limiter -> weights ->
    one-weight interpolation -> product, each step one rounding per operator"""
    lower, upper, vf = np.asarray(lower), np.asarray(upper), np.asarray(vf, float)
    F = -np.asarray(faceFlux, float) if fluxSign < 0 else np.asarray(faceFlux, float)
    lim = lo.limiter(scheme, lower, upper, F, vf, gradc, centres, k)
    w = lo.limited_weights(F, lim, np.asarray(cdWeights, float))
    r = F * (w * (vf[lower] - vf[upper]) + vf[upper])
    return -r if outSign < 0 else r


def _nhat_flux(g, S, deltaN):
    m = np.sqrt((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2])
    n = g / (m + deltaN)[:, None]
    return (n[:, 0] * S[:, 0] + n[:, 1] * S[:, 1]) + n[:, 2] * S[:, 2]


def interface_flux(lower, upper, w, gradAlpha, Sf, bFaceCells, bSf, bSnGrad, deltaN, phi=None, magSf=None, cAlpha=0.0):
    """(nHatf internal, nHatf boundary, phir or None)"""
    lower, upper = np.asarray(lower), np.asarray(upper)
    G, Sf, bSf = (np.asarray(x, float).reshape(-1, 3) for x in (gradAlpha, Sf, bSf))
    w = np.asarray(w, float)
    nHatf = _nhat_flux(w[:, None] * (G[lower] - G[upper]) + G[upper], Sf, deltaN)
    gc = G[np.asarray(bFaceCells, np.int64)]
    magS = np.sqrt((bSf[:, 0] * bSf[:, 0] + bSf[:, 1] * bSf[:, 1]) + bSf[:, 2] * bSf[:, 2])
    n = bSf / magS[:, None]
    ng = (n[:, 0] * gc[:, 0] + n[:, 1] * gc[:, 1]) + n[:, 2] * gc[:, 2]
    nHatfB = _nhat_flux(gc + n * (np.asarray(bSnGrad, float) - ng)[:, None], bSf, deltaN)
    phir = None if phi is None else (cAlpha * np.abs(np.asarray(phi, float) / np.asarray(magSf, float))) * nHatf
    return nHatf, nHatfB, phir


def delta_n(V):
    V = np.asarray(V, np.float64)
    return 1e-8 / pow(float(np.sum(V)) / len(V), 1.0 / 3.0)


class InterFoam:
    """mesh arrays + the mixture (interfaceProperties) + the fields alphaEqn.H reads and writes"""

    def __init__(self, orc, nCells, lower, upper, Sf, magSf, w, delta, V, centres, bfc, bSf, alpha1, cAlpha, sigma=0.0):
        f = lambda x: np.array(x, float)
        self.orc, self.n = orc, int(nCells)
        self.lower, self.upper = np.asarray(lower, np.int32), np.asarray(upper, np.int32)
        self.addr = orc.Addr(nCells, self.lower, self.upper)
        self.Sf, self.magSf, self.w, self.delta, self.V, self.C = f(Sf).reshape(-1, 3), f(magSf), f(w), f(delta), f(V), f(centres).reshape(-1, 3)
        self.bfc, self.bSf = np.asarray(bfc, np.int32), f(bSf).reshape(-1, 3)
        self.cAlpha, self.sigma, self.deltaN = float(cAlpha), float(sigma), delta_n(V)
        self.alpha1 = f(alpha1)
        self.alpha2 = 1.0 - self.alpha1
        self.rhoPhi = self.rhoPhiB = self.rho = None
        self.corr0 = self.corr0B = None
        self.reports = []
        self.correct()

    # ---- interfaceProperties -------------------------------------------------------------------------------------------
    def grad(self, vf):
        orc = self.orc
        face = np.asarray(orc.interpolate_linear(self.addr, self.w, vf, 1))
        return np.asarray(orc.gauss_grad(self.addr, self.Sf.ravel(), face, self.bfc, self.bSf.ravel(), vf[self.bfc], self.V, 1)).reshape(-1, 3)

    def div(self, ssf, bssf):
        return np.asarray(self.orc.surface_integrate(self.addr, ssf, self.bfc, bssf, self.V, 1, True, -1))

    def correct(self):
        self.gradAlpha = self.grad(self.alpha1)
        self.nHatf, self.nHatfB, _ = interface_flux(self.lower, self.upper, self.w, self.gradAlpha, self.Sf, self.bfc, self.bSf,
                                                    np.zeros(len(self.bfc)), self.deltaN)
        self.K = -self.div(self.nHatf, self.nHatfB)

    def surface_tension_force(self):
        orc = self.orc
        return np.asarray(orc.interpolate_linear(self.addr, self.w, self.sigma * self.K, 1)) * np.asarray(orc.sngrad(self.addr, self.delta, self.alpha1, 1))

    def near_interface(self):
        return np.where(self.alpha1 - 0.01 >= 0, 1.0, 0.0) * np.where(0.99 - self.alpha1 >= 0, 1.0, 0.0)

    # ---- alphaEqn.H ----------------------------------------------------------------------------------------------------
    def _report(self):
        self.reports.append((float((self.alpha1 * self.V).sum() / self.V.sum()), float(self.alpha1.min()), float(self.alpha1.max())))

    def alpha_eqn(self, phi, phiB, deltaT, controls, rho1, rho2, solver=("smoothSolver", "GaussSeidel"), solverControls=None):
        orc, n, l, u, bfc, V = self.orc, self.n, self.lower, self.upper, self.bfc, self.V
        phi, phiB = np.asarray(phi, float), np.asarray(phiB, float)
        aS, rS = controls["alphaScheme"], controls["alpharScheme"]
        corrected, prevCorr = bool(controls.get("MULESCorr", False)), bool(controls.get("alphaApplyPrevCorr", False))
        nIter, extrema = int(controls.get("nLimiterIter", 3)), float(controls.get("extremaCoeff", 0.0))
        rDeltaT = 1.0 / deltaT
        alpha0 = self.alpha1
        phic = self.cAlpha * np.abs(phi / self.magSf)
        phiAlpha = phiAlphaB = None
        if corrected:
            ddtDiag, ddtSource = rDeltaT * V, (rDeltaT * self.alpha1) * V
            cLower, cUpper, cDiag = (np.asarray(x) for x in orc.convection_fill(self.addr, np.where(phi >= 0, 1.0, 0.0), phi))
            eqn = fo.FvMatrix(orc, self.addr, 1, ddtDiag + cDiag, cUpper, cLower, ddtSource, self.alpha1, V, bfc, phiB[:, None],
                              np.zeros((len(bfc), 1)))
            out, _, _ = eqn.solve(solver[0], solver[1], **(solverControls or dict(tolerance=1e-8, relTol=0.0)))
            self.alpha1 = np.asarray(out).reshape(-1)
            self._report()
            eqn.psi = self.alpha1.reshape(-1, 1)
            fi, fb, _ = eqn.flux()
            UD, UDB = np.asarray(fi).reshape(-1), np.asarray(fb).reshape(-1)
            phiAlpha, phiAlphaB = UD, UDB
            if prevCorr and self.corr0 is not None:
                c0, c0B = mo.limit_corr(n, l, u, bfc, V, rDeltaT, self.alpha1, self.alpha1[bfc], phiAlphaB, self.corr0, self.corr0B, 1.0, 0.0,
                                        nIter, extremaCoeff=extrema)
                self.alpha1 = mo.correct(n, l, u, bfc, V, rDeltaT, self.alpha1, c0, c0B)
                phiAlpha, phiAlphaB = phiAlpha + c0, phiAlphaB + c0B
            self.corr0, self.corr0B = UD, UDB
            self.alpha2 = 1.0 - self.alpha1
            self.correct()
        for aCorr in range(int(controls["nAlphaCorr"])):
            phir = phic * self.nHatf
            a1B = self.alpha1[bfc]
            g1, g2 = self.gradAlpha, self.grad(self.alpha2)
            phirb = limited_flux(rS[0], l, u, phir, self.alpha2, g2, self.C, self.w, rS[1], -1, -1)
            Un = limited_flux(aS[0], l, u, phi, self.alpha1, g1, self.C, self.w, aS[1]) + \
                limited_flux(rS[0], l, u, phirb, self.alpha1, g1, self.C, self.w, rS[1])
            UnB = phiB * a1B
            if corrected:
                corr, corrB = Un - phiAlpha, UnB - phiAlphaB
                alpha10 = self.alpha1
                corr, corrB = mo.limit_corr(n, l, u, bfc, V, rDeltaT, self.alpha1, a1B, UnB, corr, corrB, 1.0, 0.0, nIter, extremaCoeff=extrema)
                self.alpha1 = mo.correct(n, l, u, bfc, V, rDeltaT, self.alpha1, corr, corrB)
                if aCorr == 0:
                    phiAlpha, phiAlphaB = phiAlpha + corr, phiAlphaB + corrB
                else:
                    self.alpha1 = 0.5 * self.alpha1 + 0.5 * alpha10
                    phiAlpha, phiAlphaB = phiAlpha + 0.5 * corr, phiAlphaB + 0.5 * corrB
            else:
                phiAlpha, phiAlphaB = mo.limit(n, l, u, bfc, V, rDeltaT, self.alpha1, alpha0, a1B, phi, phiB, Un, UnB, 1.0, 0.0, 3)
                self.alpha1 = mo.explicit_solve(n, l, u, bfc, V, rDeltaT, alpha0, phiAlpha, phiAlphaB)
            self.alpha2 = 1.0 - self.alpha1
            self.correct()
        self.rhoPhi = phiAlpha * (rho1 - rho2) + phi * rho2
        self.rhoPhiB = phiAlphaB * (rho1 - rho2) + phiB * rho2
        if prevCorr and corrected:
            self.corr0, self.corr0B = phiAlpha - self.corr0, phiAlphaB - self.corr0B
        self._report()

    def alpha_eqn_sub_cycle(self, phi, phiB, deltaT, controls, rho1, rho2, **kw):
        nSub = int(controls["nAlphaSubCycles"])
        if nSub > 1:
            sub = deltaT / nSub
            s, sB = 0.0 * np.asarray(phi, float), 0.0 * np.asarray(phiB, float)
            for _ in range(nSub):
                self.alpha_eqn(phi, phiB, sub, controls, rho1, rho2, **kw)
                s, sB = s + (sub / deltaT) * self.rhoPhi, sB + (sub / deltaT) * self.rhoPhiB
            self.rhoPhi, self.rhoPhiB = s, sB
        else:
            self.alpha_eqn(phi, phiB, deltaT, controls, rho1, rho2, **kw)
        self.rho = self.alpha1 * rho1 + self.alpha2 * rho2
