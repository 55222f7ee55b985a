"""The k-epsilon, SIMPLE and interFoam (MULESCorr) steps run in lockstep with their numpy restatements, solve by solve.

Every linear solve of these steps goes through `capi.FvMatrix.solve` on the product side and `oracle.fvm_oracle.FvMatrix.solve`
on the oracle side.  The harness wraps the two (monkeypatch, inside the test only):

 1. the product run records, per solve, the arrays of the last `LduMatrix.set` of the solved matrix (copied when `set` is
    called: the library solves with its own copies, so a later in-place `relax` must not reach the record), the FvMatrix's
    diag, source, internalCoeffs and boundaryCoeffs, solver, preconditioner, nComp, controls, psi before and after, and the
    Perf list;
 2. the oracle run, from the same starting state, checks that every system it is about to solve equals the product's record of
    the same call bit for bit (the diagonal against the MATRIX' copy, absent arrays absent on both sides, same number and
    order of solves), runs its own solve, holds the product's Perf to the Krylov contract of DESIGN.md section 2, and hands
    back the PRODUCT's solution, so that both sides go on from identical state;
 3. every solution -- the product's and, for the calibration of the bound, the oracle's own -- is checked against the system
    the oracle was given: the true residual b - A psi of every row summed exactly (each product split into two doubles that
    add up to it exactly, then math.fsum per row), normalised by the reference's normFactor (lduMatrixSolver.C:183-236)
    formed the same way.  It has to lie within TRUE_RESIDUAL_BOUND of the reported finalResidual, and at or below the
    tolerance of a solve that says it converged.  This is what catches a solve of the wrong system (a matrix not set again
    after relax) even where the oracle makes the same mistake.

Between the solves every field a step produces is compared bit for bit (int64 views: -0.0 != +0.0).  The one exception is
the volume-weighted mean of interFoam's report line, a global sum whose order differs (DESIGN.md section 2 (ii)).

The harness runs on the oracle-backed stand-in (tests/oracle_backend.py and tests/interfoam_backend.py, CPU, unmarked: it tests the harness itself and
calibrates the residual bound) and on the device (`gpu`)."""
import importlib
import math

import numpy as np
import pytest

import interfoam_backend
import interfoam_cases as ic
import polymesh_cases as pc
from oracle import fvm_oracle as fo
from oracle import kepsilon_oracle as ko
from oracle import piso_oracle as po
from test_gpu_engine_streams import Mismatches
from test_host_kernels_cpu import _d, hk  # noqa: F401  (fixture: the host build of the kernels)

BACKENDS = ["stand-in", pytest.param("device", marks=pytest.mark.gpu)]
PERF_FIELDS = ("initialResidual", "finalResidual", "normFactor", "nIterations", "converged", "singular")
SMALL = 1e-20          # solverPerformance::small_

# |true - reported| <= TRUE_RESIDUAL_BOUND for every solve: the normalised true residual of the solution against the finalResidual the
# solver reports (its recurrence residual; smoothSolver's is the true residual of its last sweep, summed in floating point).
# Measured on the CPU with the oracle's own solutions, over the 58 component solves of the stand-in cases below (PBiCG + DILU, PCG +
# DIC, smoothSolver + GaussSeidel; tolerance 1e-12, relTol 0): largest |true - reported| 6.3e-16, at a reported 7.14e-13 (the
# epsilon solve of the first upwind k-epsilon corrector); largest true residual of a converged solve 9.93e-13.  The bound keeps a
# factor of 8 over the largest difference and is 0.5 % of the tolerance: a solve of another system misses it by orders of magnitude.
TRUE_RESIDUAL_BOUND = 5e-15
# The final residuals the product and the oracle report agree to rel 1e-9 above this absolute floor (normalised).  Measured on an
# H100 80GB HBM3 (700 W limit) over the 58 component solves of the device cases: 8.2e-16 apart (rel 4e-3) for a one-iteration k
# solve whose residual falls from 0.5 to 2e-13 (the bound() edge case: a diagonal of 1e14 where k = kMin), and rel 1.5e-5
# (1e-17 apart) for SIMPLE's PCG pressure solves at 39 to 46 iterations, past the 30 iterations over which DESIGN.md section 2
# holds histories to rel 1e-9.  Both are cancellation in the recurrence residual, with the global sums in another order; every
# other solve agreed to rel 2e-11.
FINAL_RESIDUAL_FLOOR = 2e-15


@pytest.fixture(scope="module", params=BACKENDS)
def backend(request):
    if request.param == "stand-in":       # tests/oracle_backend.py with the interFoam entry points
        yield interfoam_backend.fixture()
        return
    import torch
    assert torch.cuda.is_available()
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


def host(x):
    return None if x is None else x.detach().cpu().numpy().astype(np.float64, copy=True).ravel()


def perf_of(p):
    return {k: (getattr(p, k) if k in ("initialResidual", "finalResidual", "normFactor") else int(getattr(p, k))) for k in PERF_FIELDS}


# ---- exact residuals --------------------------------------------------------------------------------------------------------------
def two_product(a, b):
    """p, e with p + e == a*b exactly (Dekker / Veltkamp splitting; exact unless a product under- or overflows)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    p = a * b
    sp = 134217729.0
    ca, cb = sp * a, sp * b
    ah, bh = ca - (ca - a), cb - (cb - b)
    al, bl = a - ah, b - bh
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def row_sums(n, rows, terms):
    """per row, the correctly rounded exact sum of the terms (math.fsum)"""
    order = np.argsort(rows, kind="stable")
    rows, terms = rows[order], terms[order]
    starts = np.searchsorted(rows, np.arange(n + 1))
    return np.array([math.fsum(terms[starts[i]:starts[i + 1]]) for i in range(n)])


def exact_Ax_minus(n, lower, upper, diag, up, low, x, b=None):
    """row sums of b - A x (b None: of A x), every product exact"""
    rows, terms = [], []
    sign = -1.0 if b is not None else 1.0
    for r, c, x_ in ((np.arange(n), diag, x), (lower, up, x[upper]), (upper, low, x[lower])):
        p, e = two_product(c, x_)
        rows += [r, r]
        terms += [sign * p, sign * e]
    if b is not None:
        rows.append(np.arange(n))
        terms.append(np.asarray(b, np.float64))
    return row_sums(n, np.concatenate(rows).astype(np.int64), np.concatenate(terms))


def solved_systems(om):
    """the diagonal and source solveSegregated hands the solver per component (fvMatrixSolve.C:104-226, fvScalarMatrix.C:142-192)
    of a single-domain fvMatrix"""
    assert not len(om.cfc), "the lockstep cases are single-domain"
    total = om.source.copy()
    om.addBoundarySource(total, False)
    out = []
    for k in range(om.nc):
        diag = om.diag.copy()
        om.addBoundaryDiag(diag, k)
        out.append((diag, np.ascontiguousarray(total[:, k])))
    return out


def true_residual(om, diag, source, psi0, psi):
    """(normalised true residual of psi, normFactor of psi0): sum |b - A psi| / normFactor, both summed exactly"""
    n, a = om.n, om.addr
    lower, upper = np.asarray(a.lower(), np.int64), np.asarray(a.upper(), np.int64)
    up, low = om.upper, om.upper if om.lower is None else om.lower
    # normFactor: sumA (row sums of the coefficients), gAverage(psi0), sum |A psi0 - sumA*avg| + |b - sumA*avg| + small
    sumA = row_sums(n, np.concatenate([np.arange(n), lower, upper]), np.concatenate([diag, up, low]))   # lduMatrixATmul.C sumA
    avg = math.fsum(psi0) / n
    Apsi0 = exact_Ax_minus(n, lower, upper, diag, up, low, psi0)
    t = avg * sumA
    normFactor = math.fsum(np.concatenate([np.abs(Apsi0 - t), np.abs(source - t)])) + SMALL
    r = exact_Ax_minus(n, lower, upper, diag, up, low, psi, source)
    return math.fsum(np.abs(r)) / normFactor, normFactor


# ---- the harness ------------------------------------------------------------------------------------------------------------------
class Lockstep:
    def __init__(self, monkeypatch, capi, device):
        self.mp, self.capi, self.device = monkeypatch, capi, device
        self.dev, self.k, self.M, self.paused = [], 0, Mismatches(), False
        self.residuals = []          # (side, solve, component, true, reported, tolerance bound, converged)

    # 1. the product run
    def record(self):
        capi, sets = self.capi, {}
        set0, solve0 = capi.LduMatrix.set, capi.FvMatrix.solve

        def set_(mat, diag, upper, lower=None, bou=None, intc=None):
            sets[mat] = tuple(host(x) for x in (diag, upper, lower, bou, intc))
            return set0(mat, diag, upper, lower, bou, intc)

        def solve(fv, solver, pre, gamg=None, pnf=None, **ctl):
            if self.paused:
                return solve0(fv, solver, pre, gamg, pnf, **ctl)
            rec = dict(set=sets[fv.m], diag=host(fv.diag), source=host(fv.source), ic=host(fv.ic), bc=host(fv.bc), solver=solver,
                       pre=pre, nc=fv.nc, ctl=dict(ctl), psi0=host(fv.psi), pnf=pnf is not None)
            perfs = solve0(fv, solver, pre, gamg, pnf, **ctl)
            rec.update(psi=host(fv.psi), perfs=[perf_of(p) for p in perfs])
            self.dev.append(rec)
            return perfs

        self.mp.setattr(capi.LduMatrix, "set", set_)
        self.mp.setattr(capi.FvMatrix, "solve", solve)

    # 2. the oracle run
    def replay(self):
        self.mp.undo()               # the stand-in's own FvMatrix is built on fo.FvMatrix: unwrap the product side first
        solve0 = fo.FvMatrix.solve

        def solve(om, solver, precond, gamg=None, pnf=None, **controls):
            i = self.k
            self.k += 1
            M = self.M
            if i >= len(self.dev):
                M.true(False, f"the oracle solves more often than the product ({i + 1} > {len(self.dev)})")
                return solve0(om, solver, precond, gamg, pnf, **controls)
            d, tag = self.dev[i], f"solve {i} ({solver} {om.nc})"
            M.true((solver, precond, om.nc, controls, pnf is not None) == (d["solver"], d["pre"], d["nc"], d["ctl"], d["pnf"]),
                   f"{tag}: solver / controls {(solver, precond, om.nc, controls)} vs {(d['solver'], d['pre'], d['nc'], d['ctl'])}")
            sDiag, sUpper, sLower, sBou, sInt = d["set"]
            M.bits(om.diag, sDiag, f"{tag}: diag vs the matrix' copy")
            M.bits(d["diag"], sDiag, f"{tag}: the FvMatrix's diag vs the matrix' copy")
            M.bits(om.upper, sUpper, f"{tag}: upper")
            M.true((om.lower is None) == (sLower is None), f"{tag}: lower present {om.lower is not None} vs {sLower is not None}")
            if om.lower is not None and sLower is not None:
                M.bits(om.lower, sLower, f"{tag}: lower")
            M.true(len(om.cfc) == 0 and sBou is None and sInt is None, f"{tag}: interface coefficients on a single domain")
            for nm, got in (("source", om.source), ("psi", om.psi), ("ic", om.ic), ("bc", om.bc)):
                M.bits(got.ravel(), d["psi0" if nm == "psi" else nm], f"{tag}: {nm}")
            psi, perfs, hists = solve0(om, solver, precond, gamg, pnf, **controls)
            self.perf_contract(tag, d["perfs"], [perf_of(p) for p in perfs])
            psiDev = d["psi"].reshape(om.n, om.nc)
            tol, relTol = controls.get("tolerance", 1e-6), controls.get("relTol", 0.0)
            for k, (diag, source) in enumerate(solved_systems(om)):
                for side, x, p in (("product", psiDev[:, k], d["perfs"][k]), ("oracle", psi[:, k], perf_of(perfs[k]))):
                    true, nf = true_residual(om, diag, source, np.ascontiguousarray(om.psi[:, k]), np.ascontiguousarray(x))
                    self.residuals.append((side, i, k, true, p["finalResidual"], max(tol, relTol * p["initialResidual"]),
                                           bool(p["converged"])))
                    M.close(p["normFactor"], nf, f"{tag}[{k}] {side}: normFactor vs the exact one", 1e-12)
            return psiDev.copy(), perfs, hists

        self.mp.setattr(fo.FvMatrix, "solve", solve)

    def perf_contract(self, tag, dev, ref):
        """DESIGN.md section 2: identical iteration counts (+-1 beyond 100), the first residual bit for bit on the stand-in and to
        rel 1e-12 on the device (global sums in another order), the final residual to rel 1e-9 above FINAL_RESIDUAL_FLOOR"""
        M = self.M
        M.true(len(dev) == len(ref), f"{tag}: {len(dev)} vs {len(ref)} components")
        for k, (p, q) in enumerate(zip(dev, ref)):
            t = f"{tag}[{k}]"
            M.true(abs(p["nIterations"] - q["nIterations"]) <= (0 if q["nIterations"] < 100 else 1),
                   f"{t}: {p['nIterations']} vs {q['nIterations']} iterations")
            M.true((p["converged"], p["singular"]) == (q["converged"], q["singular"]), f"{t}: converged / singular differ")
            if self.device:
                M.close(p["initialResidual"], q["initialResidual"], f"{t}: initialResidual", 1e-12)
            else:
                M.bits(np.ravel(p["initialResidual"]), np.ravel(q["initialResidual"]), f"{t}: initialResidual")
            if p["nIterations"] == q["nIterations"]:
                a, b = p["finalResidual"], q["finalResidual"]
                M.true(abs(a - b) <= 1e-9 * abs(b) + FINAL_RESIDUAL_FLOOR, f"{t}: finalResidual {a!r} vs {b!r}")

    # 3. and the end
    def finish(self, dev_snaps, ora_snaps):
        M = self.M
        M.true(self.k == len(self.dev), f"the product solved {len(self.dev)} times, the oracle {self.k}")
        M.true(len(dev_snaps) == len(ora_snaps), f"{len(dev_snaps)} vs {len(ora_snaps)} steps")
        for s, (a, b) in enumerate(zip(dev_snaps, ora_snaps)):
            M.true(a.keys() == b.keys(), f"step {s}: fields {sorted(a)} vs {sorted(b)}")
            for nm in a:
                if nm == "report-mean":
                    M.close(a[nm], b[nm], f"step {s}: {nm}", 1e-14)
                else:
                    M.bits(np.ravel(a[nm]), np.ravel(b[nm]), f"step {s}: {nm}")
        for side, i, k, true, reported, tol, conv in self.residuals:
            M.true(abs(true - reported) <= TRUE_RESIDUAL_BOUND,
                   f"solve {i}[{k}] {side}: true residual {true:.3e} vs reported {reported:.3e}")
            if conv:
                M.true(true <= tol, f"solve {i}[{k}] {side}: converged, true residual {true:.3e} > {tol:.1e}")
        M.true(len(self.dev) > 0, "no solve recorded")
        M.check()


def run_lockstep(monkeypatch, backend, product, oracle):
    """product(capi, ctx, torch, lockstep) and oracle() return the list of per-step snapshots {name: array}"""
    capi, ctx, torch = backend
    L = Lockstep(monkeypatch, capi, ctx.device != "cpu")
    L.record()
    dev = product(capi, ctx, torch, L)
    L.replay()
    ora = oracle()
    L.finish(dev, ora)
    L.snaps = ora
    return L


# ---- k-epsilon ----------------------------------------------------------------------------------------------------------------------
CTL = dict(tolerance=1e-12, relTol=0.0)


def _ke_snap(m, ke, host_):
    h = (lambda x: host(x)) if host_ else (lambda x: np.asarray(x, np.float64).ravel().copy())
    out = {nm: h(getattr(ke, nm)) for nm in ("k", "epsilon", "nut", "kB", "epsB", "nutB")}
    if hasattr(ke, "G"):
        out["G"] = h(ke.G)
    return out


def _edge_k(n, inner_block, kMin):
    """k for bound(): -1e-3, +0, -0, exactly kMin, denormals of both signs, a block of negative cells (its centre has only negative
    neighbours, so fvc::average(max(k, kMin)) there is kMin)"""
    rng = np.random.default_rng(11)
    k = rng.uniform(0.01, 0.02, n)
    k[:5] = -1e-3
    k[5:13] = [0.0, -0.0, kMin, 5e-324, -5e-324, 2.2250738585072009e-308, -1e-310, kMin * (1 - 2 ** -52)]
    k[inner_block] = -rng.uniform(1e-4, 1e-3, len(inner_block))
    return k


def _edge_eps(n):
    rng = np.random.default_rng(12)
    e = rng.uniform(0.05, 0.1, n)
    e[20:24] = [-0.05, -0.0, 0.0, -1e-320]
    return e


def _kepsilon_case(meshmod, orc, n=10, divScheme="upwind", alpha=None, edges=False):
    m, ref = po.cavity_from_hex(orc, meshmod, n)
    nB = len(ref.bfc)
    bMagSf, bDelta = np.full(nB, m.h * m.h), np.full(nB, 2.0 / m.h)
    kB, eB = np.full(nB, 0.015), np.full(nB, 0.08)
    ijk = lambda i, j, k: i + n * (j + n * k)
    block = np.array([ijk(i, j, k) for i in (4, 5, 6) for j in (4, 5, 6) for k in (4, 5, 6)])
    if edges:
        k0, e0 = _edge_k(m.nCells, block, ko.SMALL), _edge_eps(m.nCells)
    else:
        rng = np.random.default_rng(3)
        k0, e0 = rng.uniform(0.01, 0.02, m.nCells), rng.uniform(0.05, 0.1, m.nCells)
        k0[:5] = -1e-3
    flow = {}

    def product(capi, ctx, torch, L):
        ico = importlib.import_module("rapidcfd-dev_b200.icofoam")
        kem = importlib.import_module("rapidcfd-dev_b200.kepsilon")
        m2, case = ico.cavity(capi, ctx, torch, n)
        L.paused = True                 # the PISO steps only make the flow; the oracle side takes it as it is
        for _ in range(3):
            case.step(UControls=CTL, pControls=CTL)
        L.paused = False
        flow.update(U=host(case.U).reshape(-1, 3), phi=host(case.phi), bphi=host(case.bphi), deltaT=case.deltaT)
        ke = kem.KEpsilon(capi, case, bMagSf, bDelta, k0, e0, kB, eB)
        snaps = [_ke_snap(m, ke, True)]
        for it in range(3):
            ke.correct(case.U, case.phi, case.bphi, case.deltaT, divScheme, alpha, alpha, controls=CTL)
            snaps.append(_ke_snap(m, ke, True))
            if edges and it == 0:        # bound() on edge values after a solve, then go on from there
                ke.k, ke.kB = ke.bound(case._t(_edge_k(m.nCells, block, ke.kMin)), ke.kB, ke.kMin)
                ke.epsilon, ke.epsB = ke.bound(case._t(_edge_eps(m.nCells)), ke.epsB, ke.epsilonMin)
                snaps.append(_ke_snap(m, ke, True))
        ke.close()
        case.close()
        return snaps

    def oracle():
        ke = ko.KEpsilon(orc, ref.addr, ref.Sf, ref.magSf, ref.w, ref.delta, ref.V, ref.bfc, ref.bSf, bMagSf, bDelta, ref.Ub, ref.nu, k0, e0,
                         kB, eB)
        snaps = [_ke_snap(m, ke, False)]
        for it in range(3):
            ke.correct(flow["U"], flow["phi"], flow["bphi"], flow["deltaT"], divScheme, alpha, alpha, controls=CTL)
            snaps.append(_ke_snap(m, ke, False))
            if edges and it == 0:
                ke.k, ke.epsilon = _edge_k(m.nCells, block, ke.kMin), _edge_eps(m.nCells)
                ke.bound("k", ke.kMin)
                ke.bound("epsilon", ke.epsilonMin)
                snaps.append(_ke_snap(m, ke, False))
        return snaps

    return product, oracle, (k0, e0, block)


def _kepsilon_polymesh_case(orc):
    """k-epsilon on the split-hex box (walls only) with a prescribed velocity and a solenoidal flux, no PISO: rows with up to 24
    faces per side in fv_grad_linear, symm_magsqr, the fills and bound()"""
    b = pc.refined_box(5, "random", seed=7)
    assert b.counts()["owner"].max() >= 20 or b.counts()["losort"].max() >= 20
    C, nB = b.cell_centres(), len(b.bFaceCells)
    U, Ub, phi = pc.velocity(C), pc.velocity(b.bCf), pc.solenoidal_flux(b)
    bphi, deltaT, nu = np.zeros(nB), 0.02, 0.01
    geo = (b.nCells, b.lower, b.upper, b.Sf(), b.magSf(), b.weights(), b.deltaCoeffs(), b.volumes(), b.bFaceCells, b.bSf, b.bMagSf(),
           b.bDeltaCoeffs(), Ub, nu, deltaT)
    rng = np.random.default_rng(13)
    k0, e0 = rng.uniform(0.01, 0.02, b.nCells), rng.uniform(0.05, 0.1, b.nCells)
    k0[::17] = -1e-3
    kB, eB = np.full(nB, 0.015), np.full(nB, 0.08)

    def product(capi, ctx, torch, L):
        ico = importlib.import_module("rapidcfd-dev_b200.icofoam")
        kem = importlib.import_module("rapidcfd-dev_b200.kepsilon")
        case = ico.IcoFoam(capi, ctx, torch, *geo, cellCentres=C)
        case.U, case.phi, case.bphi = case._t(U), case._t(phi), case._t(bphi)
        ke = kem.KEpsilon(capi, case, b.bMagSf(), b.bDeltaCoeffs(), k0, e0, kB, eB)
        snaps = [_ke_snap(None, ke, True)]
        for divScheme, alpha in (("upwind", None), ("linear", 0.7), ("linear", None)):
            ke.correct(case.U, case.phi, case.bphi, deltaT, divScheme, alpha, alpha, controls=CTL)
            snaps.append(_ke_snap(None, ke, True))
        ke.close()
        case.close()
        return snaps

    def oracle():
        ref = po.Cavity(orc, *geo)
        ke = ko.KEpsilon(orc, ref.addr, ref.Sf, ref.magSf, ref.w, ref.delta, ref.V, ref.bfc, ref.bSf, b.bMagSf(), b.bDeltaCoeffs(), ref.Ub, nu,
                         k0, e0, kB, eB)
        snaps = [_ke_snap(None, ke, False)]
        for divScheme, alpha in (("upwind", None), ("linear", 0.7), ("linear", None)):
            ke.correct(U, phi, bphi, deltaT, divScheme, alpha, alpha, controls=CTL)
            snaps.append(_ke_snap(None, ke, False))
        return snaps

    return product, oracle


def _simple_case(meshmod, orc, n=8, nIter=4):
    def product(capi, ctx, torch, L):
        ico = importlib.import_module("rapidcfd-dev_b200.icofoam")
        _, dev = ico.cavity(capi, ctx, torch, n, nu=0.05)
        snaps = []
        for _ in range(nIter):
            dev.simple_step(UControls=CTL, pControls=CTL)
            snaps.append(dict(U=host(dev.U), p=host(dev.p), phi=host(dev.phi), bphi=host(dev.bphi)))
        dev.close()
        return snaps

    def oracle():
        _, ref = po.cavity_from_hex(orc, meshmod, n, nu=0.05)
        snaps = []
        for _ in range(nIter):
            ref.simple_step(UControls=CTL, pControls=CTL)
            snaps.append(dict(U=ref.U.ravel().copy(), p=ref.p.copy(), phi=ref.phi.copy(), bphi=ref.bphi.copy()))
        return snaps

    return product, oracle


def _interfoam_case(meshmod, orc, n=12, nSteps=3):
    m = meshmod.hex_mesh(n)
    a0 = ic.sphere(m)
    ctl = ic.controls(True, 2, 2)
    phi, dt = ic.rotation_flux(m)
    report = lambda r: {"report-mean": np.array(r)[:, 0].copy(), "report-min-max": np.array(r)[:, 1:].ravel()}

    def product(capi, ctx, torch, L):
        itf, mesh, mix, ph = ic.product(capi, ctx, torch, m, a0, ctl["cAlpha"])
        phiD, snaps = mesh.t(phi), []
        for _ in range(nSteps):
            itf.alpha_eqn_sub_cycle(capi, mesh, mix, ph, phiD, mesh.zeroB, dt, ctl, ic.RHO1, ic.RHO2, **ic.SOLVER)
            s = {k: host(getattr(ph, k)) for k in ("alpha1", "alpha2", "rhoPhi", "rhoPhiB", "rho")}
            s.update(K=host(mix.K), nHatf=host(mix.nHatf), nHatfB=host(mix.nHatfB), **report(ph.reports))
            snaps.append(s)
        mesh.close()
        return snaps

    def oracle():
        o, snaps = ic.oracle(orc, m, a0, ctl["cAlpha"]), []
        for _ in range(nSteps):
            o.alpha_eqn_sub_cycle(phi, np.zeros(len(o.bfc)), dt, ctl, ic.RHO1, ic.RHO2, **ic.SOLVER)
            s = {k: np.asarray(getattr(o, k), np.float64).ravel().copy() for k in ("alpha1", "alpha2", "rhoPhi", "rhoPhiB", "rho")}
            s.update(K=o.K.copy(), nHatf=o.nHatf.copy(), nHatfB=o.nHatfB.copy(), **report(o.reports))
            snaps.append(s)
        return snaps

    return product, oracle


# ---- the tests ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [None, 0.7])
@pytest.mark.parametrize("divScheme", ["upwind", "linear"])
def test_kepsilon_cavity_in_lockstep(monkeypatch, backend, meshmod, orc, divScheme, alpha):
    product, oracle, _ = _kepsilon_case(meshmod, orc, 10, divScheme, alpha)
    L = run_lockstep(monkeypatch, backend, product, oracle)
    assert len(L.dev) == 6


def test_kepsilon_bound_edge_values_in_lockstep(monkeypatch, backend, meshmod, orc):
    product, oracle, (k0, e0, block) = _kepsilon_case(meshmod, orc, 10, "upwind", 0.7, edges=True)
    L = run_lockstep(monkeypatch, backend, product, oracle)
    assert len(L.dev) == 6
    # what the edge values are there for: every neighbour of the block's centre is negative, so its bounded k is the average of
    # kMin over its faces (kMin to rounding), in the constructor and after the first solve
    centre = block[len(block) // 2]
    assert (k0[block] < 0).all() and (e0 < 0).any()
    for snap in (L.snaps[0], L.snaps[2]):
        assert snap["k"][centre] == pytest.approx(ko.SMALL, rel=1e-14) and (snap["k"] >= ko.SMALL).all()
        assert (snap["epsilon"] >= ko.SMALL).all()


def test_kepsilon_polymesh_in_lockstep(monkeypatch, backend, orc):
    product, oracle = _kepsilon_polymesh_case(orc)
    L = run_lockstep(monkeypatch, backend, product, oracle)
    assert len(L.dev) == 6


def test_simple_in_lockstep(monkeypatch, backend, meshmod, orc):
    product, oracle = _simple_case(meshmod, orc)
    L = run_lockstep(monkeypatch, backend, product, oracle)
    assert len(L.dev) == 4 * 2 and [d["nc"] for d in L.dev[:2]] == [3, 1]


def test_interfoam_mulescorr_in_lockstep(monkeypatch, backend, meshmod, orc):
    product, oracle = _interfoam_case(meshmod, orc)
    L = run_lockstep(monkeypatch, backend, product, oracle)
    assert len(L.dev) == 3 * 2


# ---- min / max follow the reference's rule ---------------------------------------------------------------------------------------
SPECIAL = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 5e-324, -5e-324, 2.2250738585072009e-308, -1e-310, 1e-15, -1e-3, 1.0,
                    1.0 + 2 ** -52, -1.0, 1e308])


def _max(s1, s2):            # label.H:285-297 (MAXMIN), instantiated for doubles by doubleFloat.H:69-86
    return s1 if s1 > s2 else s2


def _min(s1, s2):
    return s1 if s1 < s2 else s2


def _ref(f, A, B):
    return np.array([f(float(a), float(b)) for a, b in zip(A, B)])


def _host_fieldops(hk):
    """the host build of csrc/fieldops_kernels.cuh (tests/host_kernels/) behind the surface of FieldOps"""
    import ctypes as C

    class Ops:
        MIN, MAX = 4, 5

        def binary(self, op, a, b):
            out = np.zeros(len(a))
            hk.hk_field_binary(op, C.c_longlong(len(a)), 1, _d(np.ascontiguousarray(a)), 1, _d(np.ascontiguousarray(b)), _d(out))
            return out

        def _un(self, op, a, s):
            out = np.zeros(len(a))
            hk.hk_field_unary(op, C.c_longlong(len(a)), C.c_double(s), _d(np.ascontiguousarray(a)), _d(out))
            return out

        def bmax(self, a, b):
            return self.binary(self.MAX, a, b)

        def smin(self, a, s):
            return self._un(6, a, s)

        def smax(self, a, s):
            return self._un(7, a, s)

    return Ops(), np.asarray, lambda x: x


@pytest.mark.parametrize("where", ["host build", "stand-in", pytest.param("device", marks=pytest.mark.gpu)])
def test_field_min_max_follow_the_reference_rule(request, where):
    """FieldOps.bmax, smax, smin and binary(MIN) against (s1 > s2) ? s1 : s2 and (s1 < s2) ? s1 : s2, bit for bit: +-0 (the second
    operand on a tie), NaN in either position (the second operand wins whenever a comparison is false), +-inf and denormals"""
    if where == "host build":
        ops, to, back = _host_fieldops(request.getfixturevalue("hk"))
    elif where == "stand-in":
        capi, ctx, torch = interfoam_backend.fixture()
        ops, to, back = capi.FieldOps(ctx), lambda a: torch.from_numpy(np.ascontiguousarray(a)), host
    else:
        import torch
        capi = importlib.import_module("rapidcfd-dev_b200.capi")
        ctx = capi.Context(0)
        ops, to, back = capi.FieldOps(ctx), lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(ctx.device), host
    A, B = np.repeat(SPECIAL, len(SPECIAL)), np.tile(SPECIAL, len(SPECIAL))
    M = Mismatches()
    M.bits(back(ops.bmax(to(A), to(B))), _ref(_max, A, B), "bmax")
    if where != "stand-in":              # the stand-in's FieldOps has no generic binary()
        M.bits(back(ops.binary(ops.MIN, to(A), to(B))), _ref(_min, A, B), "binary(MIN)")
    for s in SPECIAL:
        M.bits(back(ops.smax(to(SPECIAL), float(s))), _ref(_max, SPECIAL, np.full(len(SPECIAL), s)), f"smax(a, {s!r})")
        M.bits(back(ops.smin(to(SPECIAL), float(s))), _ref(_min, SPECIAL, np.full(len(SPECIAL), s)), f"smin(a, {s!r})")
    # the oracle's restatement of the rule
    M.bits(fo.max_(A, B), _ref(_max, A, B), "fvm_oracle.max_")
    M.bits(fo.min_(A, B), _ref(_min, A, B), "fvm_oracle.min_")
    M.check()
    if where == "device":
        ctx.close()
