"""What a solve hands back, solver by solver, against the oracle's solve(): the solution (including which of the
two buffers a Jacobi ping-pong ends in), the counts in perf and the residual history as the caller's buffer
receives it -- entries up to the count, NaN after it, clamped to the buffer's capacity -- and that a refused
selection leaves psi and the history buffer untouched."""
import ctypes as C
import importlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SENTINEL = 7.0


@pytest.fixture(scope="module")
def gpu():
    import torch
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


@pytest.fixture(scope="module")
def systems(gpu, meshmod, orc):
    """A symmetric (pressure) and an asymmetric (momentum) system on one mesh, on both sides."""
    capi, ctx, torch = gpu
    m = meshmod.hex_mesh(14, 12, 10)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(ctx.device)
    oa = orc.Addr(m.nCells, m.lower, m.upper)
    addr = capi.mesh_to_device(ctx, m, with_centres=True)
    xs = meshmod.cell_field_global(m, 42)
    out = {}
    for kind, c in (("P", meshmod.pressure_laplacian(m)), ("U", meshmod.momentum_matrix(m))):
        lower = c.get("lower")
        om = orc.Matrix(oa, c["diag"], c["upper"], lower)
        mat = capi.LduMatrix(addr)
        mat.set(t(c["diag"]), t(c["upper"]), t(lower) if lower is not None and len(lower) else None)
        b = om.amul(xs)
        out[kind] = dict(om=om, mat=mat, b=b, bd=t(b), diag=c["diag"])
    out["mesh"], out["oa"], out["addr"], out["t"] = m, oa, addr, t
    yield out
    for kind in ("P", "U"):
        out[kind]["mat"].close()
    addr.close()


def raw_solve(capi, torch, mat, solver, pre, psi, bd, histCap, gamg=None, **ctl):
    """b200ldu_solve with the caller's history buffer exactly as the library leaves it (pre-filled with SENTINEL)."""
    c = capi.controls(**ctl)
    perf = capi.Perf()
    hist = np.full(histCap, SENTINEL)
    rc = capi.lib().b200ldu_solve(mat.h, solver.encode(), (pre or "").encode(), C.byref(c),
                                  gamg.h if gamg is not None else None, capi._dp(psi), capi._dp(bd),
                                  C.byref(perf), capi._hp(hist), histCap)
    torch.cuda.synchronize()
    return rc, perf, hist


def check_history(hist, k, href, rtol):
    """k entries that follow the oracle, then NaN up to the capacity"""
    assert np.all(np.isfinite(hist[:k]))
    assert np.all(np.isnan(hist[k:]))
    assert len(href) >= k
    np.testing.assert_allclose(hist[:k], href[:k], rtol=rtol)


def pbicgstab_early_tolerance(om, b, n0):
    """A tolerance at which the oracle's PBiCGStab leaves at the check on s (PBiCGStab.C:198-213): its last
    history entry is then |s| / normFactor, which differs from the full-iteration residual at that count.  Any
    tolerance in (|s| / normFactor, tol] leaves at the same check; the geometric mean keeps a margin on both sides."""
    _, _, full = om.solve("PBiCGStab", "diagonal", np.zeros(n0), b, tolerance=0.0, maxIter=60)
    for tol in np.geomspace(full[1], full[-1], 400):
        _, pr, h = om.solve("PBiCGStab", "diagonal", np.zeros(n0), b, tolerance=float(tol), maxIter=60)
        k = pr.nIterations
        if pr.converged and 0 < k < len(full) and h[k] != full[k]:
            return float(np.sqrt(h[k] * tol))
    pytest.fail("no tolerance in the scan ends PBiCGStab at the check on s")


@pytest.mark.parametrize("solver,ctl", [
    ("PBiCG", dict(tolerance=1e-9, maxIter=200)),
    ("PBiCG", dict(tolerance=0.0, maxIter=7)),
    ("PBiCGStab", dict(tolerance=1e-9, maxIter=200)),
    ("PBiCGStab", dict(tolerance=1e-9, maxIter=200, bicgstabRefQuirk=1)),
    ("PBiCGStab", dict(tolerance=0.0, maxIter=7)),
    ("PBiCGStab", "early"),
])
def test_asymmetric_krylov_history(gpu, systems, solver, ctl):
    capi, ctx, torch = gpu
    s, n = systems["U"], systems["mesh"].nCells
    if ctl == "early":
        ctl = dict(tolerance=pbicgstab_early_tolerance(s["om"], s["b"], n), maxIter=60)
    psi_ref, pr, href = s["om"].solve(solver, "diagonal", np.zeros(n), s["b"], **ctl)
    psi = torch.zeros(n, dtype=torch.float64, device=ctx.device)
    rc, perf, hist = raw_solve(capi, torch, s["mat"], solver, "diagonal", psi, s["bd"], 256, **ctl)
    assert rc == 0
    assert perf.solverName == ("diagonal" + solver).encode()
    assert (perf.nIterations, perf.converged, perf.singular) == (pr.nIterations, pr.converged, pr.singular)
    assert len(href) == pr.nIterations + 1
    check_history(hist, perf.nIterations + 1, href, 1e-9)
    np.testing.assert_allclose(psi.cpu().numpy(), psi_ref, rtol=0, atol=1e-9)


@pytest.mark.parametrize("nSweeps", [1, 2, 3])
def test_smooth_solver_history(gpu, systems, nSweeps):
    capi, ctx, torch = gpu
    s, n = systems["P"], systems["mesh"].nCells
    ctl = dict(tolerance=0.0, maxIter=20, nSweeps=nSweeps)
    psi_ref, pr, href = s["om"].solve("smoothSolver", "GaussSeidel", np.zeros(n), s["b"], **ctl)
    psi = torch.zeros(n, dtype=torch.float64, device=ctx.device)
    rc, perf, hist = raw_solve(capi, torch, s["mat"], "smoothSolver", "GaussSeidel", psi, s["bd"], 64, **ctl)
    assert rc == 0
    assert perf.nIterations == pr.nIterations
    k = perf.nIterations // nSweeps + 1
    assert len(href) == k
    check_history(hist, k, href, 1e-12)
    # the buffer psi ends in: one sweep more or less would move it by far more than this
    np.testing.assert_allclose(psi.cpu().numpy(), psi_ref, rtol=0, atol=1e-12)


def test_smooth_solver_fixed_sweeps(gpu, systems):
    capi, ctx, torch = gpu
    s, m = systems["P"], systems["mesh"]
    psi_ref, pr, href = s["om"].solve("smoothSolver", "Jacobi", np.zeros(m.nCells), s["b"], nSweeps=-3)
    assert (pr.nIterations, pr.converged, len(href)) == (3, 0, 0)
    psi = torch.zeros(m.nCells, dtype=torch.float64, device=ctx.device)
    rc, perf, hist = raw_solve(capi, torch, s["mat"], "smoothSolver", "Jacobi", psi, s["bd"], 16, nSweeps=-3)
    assert rc == 0
    assert (perf.nIterations, perf.converged, perf.singular) == (3, 0, 0)
    assert np.all(np.isnan(hist))
    np.testing.assert_allclose(psi.cpu().numpy(), psi_ref, rtol=0, atol=1e-12)


def test_diagonal_solver(gpu, systems):
    capi, ctx, torch = gpu
    s, n = systems["P"], systems["mesh"].nCells
    psi_ref, pr, href = s["om"].solve("diagonal", None, np.zeros(n), s["b"])
    assert (pr.converged, len(href)) == (1, 0)
    psi = torch.zeros(n, dtype=torch.float64, device=ctx.device)
    rc, perf, hist = raw_solve(capi, torch, s["mat"], "diagonal", None, psi, s["bd"], 16)
    assert rc == 0
    assert perf.solverName == b"diagonal"
    assert (perf.nIterations, perf.converged, perf.singular) == (0, 1, 0)
    assert (perf.initialResidual, perf.finalResidual, perf.normFactor) == (0.0, 0.0, 0.0)
    assert np.all(np.isnan(hist))
    assert np.array_equal(psi.cpu().numpy(), psi_ref)


@pytest.mark.parametrize("nFinestSweeps", [1, 2, 3])
@pytest.mark.parametrize("ctl", [dict(tolerance=0.0, maxIter=3), dict(tolerance=1e-8, maxIter=100)])
def test_gamg_history_and_buffer(gpu, systems, meshmod, orc, nFinestSweeps, ctl):
    capi, ctx, torch = gpu
    s, m = systems["P"], systems["mesh"]
    w = meshmod.face_area_pair_weights(m)
    og = orc.Gamg(systems["oa"], w, 10)
    gg = capi.GamgAgglomeration(systems["addr"], w, 10)
    ctl = dict(ctl, nFinestSweeps=nFinestSweeps)
    psi_ref, pr, href = og.solve(s["om"], "GaussSeidel", np.zeros(m.nCells), s["b"], **ctl)
    psi = torch.zeros(m.nCells, dtype=torch.float64, device=ctx.device)
    rc, perf, hist = raw_solve(capi, torch, s["mat"], "GAMG", "GaussSeidel", psi, s["bd"], 256, gamg=gg, **ctl)
    gg.close()
    assert rc == 0
    assert (perf.nIterations, perf.converged) == (pr.nIterations, pr.converged)
    assert len(href) == pr.nIterations + 1
    check_history(hist, perf.nIterations + 1, href, 1e-8)
    # an odd number of finest sweeps leaves psi in the other buffer after an odd number of cycles
    np.testing.assert_allclose(psi.cpu().numpy(), psi_ref, rtol=0, atol=1e-9)


@pytest.mark.parametrize("solver,pre,kind,ctl", [
    ("PCG", "DIC", "P", dict(tolerance=0.0, maxIter=20)),
    ("PBiCGStab", "DILU", "U", dict(tolerance=0.0, maxIter=20)),
    ("smoothSolver", "Jacobi", "P", dict(tolerance=0.0, maxIter=30, nSweeps=2)),
])
def test_history_clamped_to_capacity(gpu, systems, solver, pre, kind, ctl):
    capi, ctx, torch = gpu
    s, n = systems[kind], systems["mesh"].nCells
    _, pr, href = s["om"].solve(solver, pre, np.zeros(n), s["b"], **ctl)
    cap = 5
    assert len(href) > cap
    psi = torch.zeros(n, dtype=torch.float64, device=ctx.device)
    rc, perf, hist = raw_solve(capi, torch, s["mat"], solver, pre, psi, s["bd"], cap, **ctl)
    assert rc == 0
    assert perf.nIterations == pr.nIterations
    assert len(hist) == cap and np.all(np.isfinite(hist))
    np.testing.assert_allclose(hist, href[:cap], rtol=1e-9)


@pytest.mark.parametrize("solver,pre,kind,rc", [
    ("noSuchSolver", None, "P", -3),           # B200LDU_ENOSOLVER
    ("PCG", "noSuchPreconditioner", "P", -4),  # B200LDU_ENOPRECOND
    ("PCG", "DILU", "P", -4),
    ("PBiCG", "DIC", "U", -4),
    ("PCG", "DIC", "U", -5),                   # B200LDU_EMATRIX
    ("PBiCGStab", None, "P", -5),
    ("smoothSolver", "DIC", "P", -4),
    ("GAMG", "GaussSeidel", "P", -1),          # B200LDU_EINVAL: no agglomeration handle
])
def test_refused_selection_changes_nothing(gpu, systems, solver, pre, kind, rc):
    capi, ctx, torch = gpu
    s, m = systems[kind], systems["mesh"]
    psi0 = systems["t"](0.5 + 0.25 * np.sin(np.arange(m.nCells, dtype=np.float64)))
    psi = psi0.clone()
    got, perf, hist = raw_solve(capi, torch, s["mat"], solver, pre, psi, s["bd"], 8)
    assert got == rc, capi.lib().b200ldu_last_error()
    assert torch.equal(psi, psi0)
    assert np.all(hist == SENTINEL)
