"""Cases shared by tests/test_interfoam_cpu.py, tests/test_gpu_interfoam.py and tests/golden/make_interfoam_golden.py: a cube of
N^3 cells with walls (alpha1 zeroGradient, no flux through the boundary), a smoothed sphere of alpha1 = 1 and a discretely
solenoidal rotating flux (differences of a stream function that vanishes on the walls)."""
import importlib

import numpy as np


def geometry(m):
    walls = m.wall_patches()
    return dict(nCells=m.nCells, lower=m.lower, upper=m.upper, Sf=m.Sf(), magSf=m.magSf(), weights=m.weights(), deltaCoeffs=m.deltaCoeffs(),
                V=m.volumes(), centres=m.cell_centres(), bFaceCells=np.concatenate([p.faceCells for p in walls]).astype(np.int32),
                bSf=np.concatenate([p.Sf for p in walls]))


def sphere(m, centre=(0.5, 0.3, 0.5), R=0.18, width=1.0):
    """alpha1 = 1 inside, smoothed over `width` cells"""
    r = np.sqrt(((m.cell_centres() - np.array(centre)) ** 2).sum(1))
    return 0.5 * (1.0 - np.tanh((r - R) / (width * m.h)))


def rotation_flux(m):
    """(phi on the internal faces, time step of Courant number 0.25)"""
    N, h = m.nx, m.h
    S = lambda x, y: (np.sin(np.pi * x) * np.sin(np.pi * y)) ** 2 / np.pi
    i, j = m.lower % N, (m.lower // N) % N
    phix = (S((i + 1) * h, (j + 1) * h) - S((i + 1) * h, j * h)) * h
    phiy = -(S((i + 1) * h, (j + 1) * h) - S(i * h, (j + 1) * h)) * h
    phi = np.where(m.faceDir == 0, phix, np.where(m.faceDir == 1, phiy, 0.0))
    return phi, 0.25 * h / (np.abs(phi).max() / h / h)


def controls(MULESCorr=False, nAlphaCorr=1, nAlphaSubCycles=1, cAlpha=1.0, alphaScheme=("vanLeer", 1.0), alpharScheme=("linear", 1.0),
             alphaApplyPrevCorr=False):
    return dict(MULESCorr=MULESCorr, nAlphaCorr=nAlphaCorr, nAlphaSubCycles=nAlphaSubCycles, cAlpha=cAlpha, alphaScheme=alphaScheme,
                alpharScheme=alpharScheme, alphaApplyPrevCorr=alphaApplyPrevCorr, nLimiterIter=3, extremaCoeff=0.0, icAlpha=0.0)


RHO1, RHO2 = 1000.0, 1.0
SOLVER = dict(solver=("smoothSolver", "GaussSeidel"), solverControls=dict(tolerance=1e-12, relTol=0.0, maxIter=200))


def product(capi, ctx, torch, m, alpha1, cAlpha):
    """(interfoam module, Mesh, InterfaceProperties, Phase) over capi -- the CUDA library or the stand-in"""
    itf = importlib.import_module("rapidcfd-dev_b200.interfoam")
    mesh = itf.Mesh(capi, ctx, torch, **geometry(m))
    ph = itf.Phase(mesh, np.asarray(alpha1, float))
    return itf, mesh, itf.InterfaceProperties(capi, mesh, ph.alpha1, cAlpha, 0.07), ph


def oracle(orc, m, alpha1, cAlpha):
    from oracle import interfoam_oracle as io
    g = geometry(m)
    return io.InterFoam(orc, g["nCells"], g["lower"], g["upper"], g["Sf"], g["magSf"], g["weights"], g["deltaCoeffs"], g["V"], g["centres"],
                        g["bFaceCells"], g["bSf"], alpha1, cAlpha, 0.07)


def run_product(capi, ctx, torch, m, alpha1, ctl, nSteps, kw=None):
    itf, mesh, mix, ph = product(capi, ctx, torch, m, alpha1, ctl["cAlpha"])
    phi, dt = rotation_flux(m)
    phiD = mesh.t(phi)
    for _ in range(nSteps):
        itf.alpha_eqn_sub_cycle(capi, mesh, mix, ph, phiD, mesh.zeroB, dt, ctl, RHO1, RHO2, **(kw or {}))
    return mesh, mix, ph


def run_oracle(orc, m, alpha1, ctl, nSteps, kw=None):
    o = oracle(orc, m, alpha1, ctl["cAlpha"])
    phi, dt = rotation_flux(m)
    for _ in range(nSteps):
        o.alpha_eqn_sub_cycle(phi, np.zeros(len(o.bfc)), dt, ctl, RHO1, RHO2, **(kw or {}))
    return o


def band(alpha):
    return int(((alpha > 0.01) & (alpha < 0.99)).sum())
