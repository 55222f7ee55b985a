"""The phase-fraction step of interFoam sequenced over the C ABI (host side: sequencing only, every field stays on the device):
the interface normal flux and curvature, the limited and compressive fluxes, and the alphaEqn corrector loop over explicit MULES
and CMULES.  `capi` is rapidcfd-dev_b200.capi (or, in CPU dry runs of the sequencing, an oracle-backed stand-in with the same
surface).

  alphaEqn.H, alphaEqnSubCycle.H   applications/solvers/multiphase/interFoam/
  interfaceProperties              src/transportModels/interfaceProperties/interfaceProperties.C:118-159 (calculateK), :181-185
                                   (deltaN), :220-232 (surfaceTensionForce, nearInterface)
  alphaControls                    FV/cfdTools/general/include/alphaControls.H
  MULES::explicitSolve / correct   FV/fvMatrices/solvers/MULES/MULESTemplates.C:81-115 (three limiter sweeps, fixed),
                                   CMULESTemplates.C:78-112 (nLimiterIter from the solver dictionary) -- rapidcfd-dev_b200/mules.py
The three fvc::flux of a limited scheme per corrector are one b200ldu_fv_limited_flux each; nHatf and phir come from
b200ldu_vof_interface_flux.

Scope: static mesh, single domain, alpha1 zeroGradient on every boundary face (walls).  icAlpha > 0, the LTS variants, contact
angles, moving meshes and coupled patches are refused by name (`refuse_unsupported`).  The momentum and p_rgh equations of
interFoam are not here."""
import numpy as np

from . import mules

SCHEMES = ("Minmod", "limitedLinear", "linear", "upwind", "vanLeer")


def refuse_unsupported(controls, alphaPatchTypes=(), ddtScheme="Euler", movingMesh=False, nCoupledFaces=0):
    """what this step does not do, by name; `controls`: foamfile.alpha_controls (or a dict with the same keys)"""
    if controls.get("icAlpha", 0.0) > 0:
        raise NotImplementedError(f"alpha controls: icAlpha {controls['icAlpha']} -- this step implements the standard face-flux "
                                  "compression only (icAlpha 0; alphaEqn.H:9-13)")
    if ddtScheme == "localEuler":
        raise NotImplementedError("fvSchemes: ddtSchemes localEuler -- the LTSSOLVE variants of alphaEqn.H (MULES::explicitLTSSolve, "
                                  "MULES::LTScorrect) are not implemented; this step implements Euler")
    if ddtScheme != "Euler":
        raise NotImplementedError(f"fvSchemes: ddtSchemes {ddtScheme} -- alphaEqn.H builds fv::EulerDdtScheme; this step implements Euler")
    for t in alphaPatchTypes:
        if t in ("constantAlphaContactAngle", "dynamicAlphaContactAngle", "timeVaryingAlphaContactAngle",
                 "temperatureDependentAlphaContactAngle", "alphaContactAngle"):
            raise NotImplementedError(f"alpha boundary condition {t} -- contact angles (interfaceProperties::correctContactAngle) "
                                      "are not implemented")
        if t != "zeroGradient":
            raise NotImplementedError(f"alpha boundary condition {t} -- this step supports zeroGradient")
    if movingMesh:
        raise NotImplementedError("moving mesh -- this step is for static meshes (no mesh.Vsc0(), no meshPhi)")
    if nCoupledFaces:
        raise NotImplementedError("coupled (processor / cyclic) patches -- this step runs on a single domain")
    for key in ("alphaScheme", "alpharScheme"):
        if key in controls and controls[key][0] not in SCHEMES:
            raise ValueError(f"Unknown discretisation scheme {controls[key][0]}\n\nValid schemes are :\n({' '.join(SCHEMES)})")


class Mesh:
    """the mesh arrays of one single-domain case on the device; boundary faces in patch order (all non-coupled)"""

    def __init__(self, capi, ctx, torch, nCells, lower, upper, Sf, magSf, weights, deltaCoeffs, V, centres, bFaceCells, bSf, addr=None):
        self.capi, self.ctx, self.torch = capi, ctx, torch
        self.n, self.nF = int(nCells), len(lower)
        self.addr = addr if addr is not None else capi.LduAddressing(ctx, nCells, lower, upper, cellCentres=centres)
        bfc = np.ascontiguousarray(bFaceCells, dtype=np.int32)
        self.nB = len(bfc)
        capi.fv_boundary_set(self.addr, bfc)
        self.ops = capi.FieldOps(ctx)
        t = self.t
        self.Sf, self.magSf, self.w, self.delta, self.V, self.C, self.bSf = (t(x) for x in (Sf, magSf, weights, deltaCoeffs, V, centres, bSf))
        self.bfc = torch.from_numpy(bfc.copy()).to(ctx.device)
        self.zeroB = t(np.zeros(self.nB))
        # deltaN = 1e-8/pow(average(V), 1/3) (interfaceProperties.C:181-185): a constant of the mesh, formed once on the host
        Vh = np.asarray(V, np.float64)
        self.deltaN = 1e-8 / pow(float(np.sum(Vh)) / len(Vh), 1.0 / 3.0)

    def t(self, a):
        return self.torch.from_numpy(np.array(a, dtype=np.float64).ravel()).to(self.ctx.device)

    def grad(self, vf, vfB):
        """fvc::grad, Gauss linear"""
        return self.capi.fv_grad_linear(self.addr, 1, self.Sf, self.w, vf, self.bSf, vfB, self.V)

    def close(self):
        self.addr.close()


class InterfaceProperties:
    """interfaceProperties (and, for the step, the mixture): nHatf, K, deltaN; alpha1 zeroGradient at the boundary"""

    def __init__(self, capi, mesh, alpha1, cAlpha, sigma):
        self.capi, self.mesh, self.ops = capi, mesh, mesh.ops
        self.cAlpha, self.sigma, self.deltaN = float(cAlpha), float(sigma), mesh.deltaN
        self.correct(alpha1)

    def correct(self, alpha1):
        """calculateK: gradAlpha = fvc::grad(alpha1), nHatf = nHatfv & Sf, K = -fvc::div(nHatf)"""
        capi, m, o = self.capi, self.mesh, self.ops
        self.alpha1 = alpha1
        self.gradAlpha = m.grad(alpha1, o.gather(m.bfc, alpha1))
        self.nHatf, self.nHatfB, _ = capi.vof_interface_flux(m.addr, m.w, self.gradAlpha, m.Sf, m.bSf, m.zeroB, self.deltaN)
        self.K = o.neg(capi.fv_surface_integrate(m.addr, 1, self.nHatf, self.nHatfB, m.V, True, -1))

    def compression_flux(self, phi):
        """phir = phic*nHatf on the internal faces, phic = cAlpha*mag(phi/magSf) (alphaEqn.H:6, :82); zero on the boundary faces
        (:17-25).  nHatf is formed again from the gradient of the last correct(), in the same pass."""
        m = self.mesh
        return self.capi.vof_interface_flux(m.addr, m.w, self.gradAlpha, m.Sf, m.bSf, m.zeroB, self.deltaN, phi, m.magSf, self.cAlpha)[2]

    def surface_tension_force(self):
        """fvc::interpolate(sigma*K)*fvc::snGrad(alpha1) on the internal faces"""
        capi, m, o = self.capi, self.mesh, self.ops
        return o.mul(capi.fv_interpolate_linear(m.addr, 1, m.w, o.smul(self.sigma, self.K)), capi.fv_sngrad(m.addr, 1, m.delta, self.alpha1))

    def near_interface(self):
        """pos(alpha1 - 0.01)*pos(0.99 - alpha1)"""
        o = self.ops
        return o.mul(o.pos(o.sadd(self.alpha1, -0.01)), o.pos(o.rsub(0.99, self.alpha1)))


class Phase:
    """what alphaEqn.H reads and writes: alpha1, alpha2, rhoPhi (internal and boundary faces), rho, and the cached flux of
    alphaApplyPrevCorr; `reports` collects the figures of the "Phase-1 volume fraction" lines"""

    def __init__(self, mesh, alpha1):
        self.alpha1 = mesh.t(alpha1) if isinstance(alpha1, np.ndarray) else alpha1
        self.alpha2 = mesh.ops.rsub(1.0, self.alpha1)
        self.rhoPhi = self.rhoPhiB = self.rho = None
        self.phiAlphaCorr0 = self.phiAlphaCorr0B = None
        self.reports = []


def _report(mesh, ph):
    """alpha1.weightedAverage(V), min(alpha1), max(alpha1): reductions on the device, three numbers to the host"""
    a, V = ph.alpha1, mesh.V
    r = (float((a * V).sum() / V.sum()), float(a.min()), float(a.max()))
    ph.reports.append(r)
    return "Phase-1 volume fraction = %g  Min(alpha1) = %g  Max(alpha1) = %g" % r


def _needs_grad(scheme):
    return scheme[0] not in ("upwind", "linear")


def alpha_eqn(capi, mesh, mixture, ph, phi, phiB, deltaT, controls, rho1, rho2, solver=("smoothSolver", "GaussSeidel"),
              solverControls=None, info=None):
    """alphaEqn.H, statement by statement, on `ph` (a Phase).  controls: nAlphaCorr, cAlpha (held by the mixture), MULESCorr,
    alphaApplyPrevCorr, nLimiterIter, extremaCoeff, alphaScheme / alpharScheme = (scheme word, k) of div(phi,alpha) /
    div(phirb,alpha).  solver / solverControls: the alpha solver entry of fvSolution for the MULESCorr predictor.  The mixture has
    been corrected for ph.alpha1 (as it is after every corrector)."""
    m, o, a = mesh, mesh.ops, mesh.addr
    say = info or (lambda s: None)
    aS, rS = controls["alphaScheme"], controls["alpharScheme"]
    corrected, prevCorr = bool(controls.get("MULESCorr", False)), bool(controls.get("alphaApplyPrevCorr", False))
    nIter, extrema = int(controls.get("nLimiterIter", 3)), float(controls.get("extremaCoeff", 0.0))
    rDeltaT = 1.0 / deltaT
    alpha0 = ph.alpha1                                      # alpha1.oldTime()
    bval = lambda f: o.gather(m.bfc, f)                     # zeroGradient boundary values
    phiAlpha = phiAlphaB = None
    if corrected:
        # fv::EulerDdtScheme(mesh).fvmDdt(alpha1) + fv::gaussConvectionScheme(mesh, phi, upwind(mesh, phi)).fvmDiv(phi, alpha1)
        ddtDiag, ddtSource = o.smul(rDeltaT, m.V), o.mul(o.smul(rDeltaT, ph.alpha1), m.V)
        cLower, cUpper, cDiag = capi.fv_convection_fill(a, capi.fv_limited_weights(m.ctx, phi), phi)
        diag = o.add(ddtDiag, cDiag)
        mat = capi.LduMatrix(a)
        mat.set(diag, cUpper, cLower)
        new = ph.alpha1.clone()
        eqn = capi.FvMatrix(mat, 1, diag, ddtSource, new, m.V, phiB, m.zeroB)   # zeroGradient: patchFlux*1, -patchFlux*0
        eqn.solve(solver[0], solver[1], **(solverControls or dict(tolerance=1e-8, relTol=0.0)))
        ph.alpha1 = new
        say(_report(m, ph))
        phiAlphaUD, phiAlphaUDB, _ = eqn.flux(m.nB)
        phiAlphaUDB = phiAlphaUDB[: m.nB]
        mat.close()
        phiAlpha, phiAlphaB = phiAlphaUD, phiAlphaUDB
        if prevCorr and ph.phiAlphaCorr0 is not None:
            say("Applying the previous iteration compression flux")
            c0, c0B = mules.limit_corr(capi, a, o, m.V, rDeltaT, ph.alpha1, bval(ph.alpha1), phiAlphaB, ph.phiAlphaCorr0, ph.phiAlphaCorr0B,
                                       1.0, 0.0, nIter, extremaCoeff=extrema)
            ph.alpha1 = mules.correct(capi, a, o, m.V, rDeltaT, ph.alpha1, c0, c0B)
            phiAlpha, phiAlphaB = o.add(phiAlpha, c0), o.add(phiAlphaB, c0B)
        ph.phiAlphaCorr0, ph.phiAlphaCorr0B = phiAlphaUD, phiAlphaUDB       # cache the upwind flux
        ph.alpha2 = o.rsub(1.0, ph.alpha1)
        mixture.correct(ph.alpha1)
    for aCorr in range(int(controls["nAlphaCorr"])):
        phir = mixture.compression_flux(phi)
        alpha1B = bval(ph.alpha1)
        g1 = mixture.gradAlpha if _needs_grad(aS) or _needs_grad(rS) else None       # fvc::grad(alpha1), as calculateK formed it
        g2 = m.grad(ph.alpha2, bval(ph.alpha2)) if _needs_grad(rS) else None
        # fvc::flux(phi, alpha1, alphaScheme) + fvc::flux(-fvc::flux(-phir, alpha2, alpharScheme), alpha1, alpharScheme)
        phirb = capi.fv_limited_flux(a, rS[0], phir, ph.alpha2, g2, m.C, m.w, rS[1], fluxSign=-1, outSign=-1)
        phiAlphaUn = o.add(capi.fv_limited_flux(a, aS[0], phi, ph.alpha1, g1, m.C, m.w, aS[1]),
                           capi.fv_limited_flux(a, rS[0], phirb, ph.alpha1, g1, m.C, m.w, rS[1]))
        phiAlphaUnB = o.mul(phiB, alpha1B)                  # phir is zero on the boundary faces
        if corrected:
            corr, corrB = o.sub(phiAlphaUn, phiAlpha), o.sub(phiAlphaUnB, phiAlphaB)
            alpha10 = ph.alpha1
            # MULES::correct(alpha1, tphiAlphaUn(), tphiAlphaCorr(), 1, 0): limitCorr, then correct
            corr, corrB = mules.limit_corr(capi, a, o, m.V, rDeltaT, ph.alpha1, alpha1B, phiAlphaUnB, corr, corrB, 1.0, 0.0, nIter,
                                           extremaCoeff=extrema)
            ph.alpha1 = mules.correct(capi, a, o, m.V, rDeltaT, ph.alpha1, corr, corrB)
            if aCorr == 0:
                phiAlpha, phiAlphaB = o.add(phiAlpha, corr), o.add(phiAlphaB, corrB)
            else:   # under-relax the correction for all but the first corrector
                ph.alpha1 = o.add(o.smul(0.5, ph.alpha1), o.smul(0.5, alpha10))
                phiAlpha, phiAlphaB = o.add(phiAlpha, o.smul(0.5, corr)), o.add(phiAlphaB, o.smul(0.5, corrB))
        else:
            # MULES::explicitSolve(alpha1, phi, tphiAlpha(), 1, 0): limit with three sweeps, then explicitSolve
            phiAlpha, phiAlphaB = mules.limit(capi, a, o, m.V, rDeltaT, ph.alpha1, alpha0, alpha1B, phi, phiB, phiAlphaUn, phiAlphaUnB,
                                              1.0, 0.0, 3)
            ph.alpha1 = mules.explicit_solve(capi, a, o, m.V, rDeltaT, alpha0, phiAlpha, phiAlphaB)
        ph.alpha2 = o.rsub(1.0, ph.alpha1)
        mixture.correct(ph.alpha1)
    # rhoPhi = tphiAlpha()*(rho1 - rho2) + phi*rho2
    ph.rhoPhi = o.add(o.smul(rho1 - rho2, phiAlpha), o.smul(rho2, phi))
    ph.rhoPhiB = o.add(o.smul(rho1 - rho2, phiAlphaB), o.smul(rho2, phiB))
    if prevCorr and corrected:
        ph.phiAlphaCorr0, ph.phiAlphaCorr0B = o.sub(phiAlpha, ph.phiAlphaCorr0), o.sub(phiAlphaB, ph.phiAlphaCorr0B)
    say(_report(m, ph))
    return ph


def alpha_eqn_sub_cycle(capi, mesh, mixture, ph, phi, phiB, deltaT, controls, rho1, rho2, **kw):
    """alphaEqnSubCycle.H: nAlphaSubCycles passes of alphaEqn.H over deltaT/nAlphaSubCycles with rhoPhi accumulated by the
    fraction of the time step, then rho = alpha1*rho1 + alpha2*rho2"""
    o = mesh.ops
    nSub = int(controls["nAlphaSubCycles"])
    if nSub > 1:
        sub = deltaT / nSub
        rhoPhiSum, rhoPhiSumB = o.smul(0.0, phi), o.smul(0.0, phiB)
        for _ in range(nSub):
            alpha_eqn(capi, mesh, mixture, ph, phi, phiB, sub, controls, rho1, rho2, **kw)
            rhoPhiSum, rhoPhiSumB = o.add(rhoPhiSum, o.smul(sub / deltaT, ph.rhoPhi)), o.add(rhoPhiSumB, o.smul(sub / deltaT, ph.rhoPhiB))
        ph.rhoPhi, ph.rhoPhiB = rhoPhiSum, rhoPhiSumB
    else:
        alpha_eqn(capi, mesh, mixture, ph, phi, phiB, deltaT, controls, rho1, rho2, **kw)
    ph.rho = o.add(o.smul(rho1, ph.alpha1), o.smul(rho2, ph.alpha2))
    return ph
