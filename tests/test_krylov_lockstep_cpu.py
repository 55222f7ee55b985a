"""The lockstep machinery of tests/test_gpu_krylov_lockstep.py, rehearsed on the CPU.

* The oracle's reduction hook moves nothing when it hands the oracle its own sums: every solver and preconditioner
  reproduces its unhooked run bit for bit.
* A stand-in "device" is the oracle with the device's AINV association and every global sum recomputed in numpy's
  pairwise order.  A second, hooked oracle run fed those sums matches it bit for bit after every iteration, and
  every sum passes the bound of krylov_lockstep.
* A stand-in whose search direction is one ulp off in one row at one iteration fails the comparison, and the report
  names that iteration; a stand-in whose sum drops one term fails the bound, named by site and iteration."""
import numpy as np
import pytest

import krylov_lockstep as kl

PCG_PRE = ("none", "diagonal", "DIC")
ASYM_PRE = ("none", "diagonal", "DILU")
CONFIGS = ([("PCG", p, {}) for p in PCG_PRE] + [("PBiCG", p, {}) for p in ASYM_PRE] +
           [("PBiCGStab", p, {"bicgstabRefQuirk": q}) for p in ASYM_PRE for q in (0, 1)] +
           [("smoothSolver", "GaussSeidel", {"nSweeps": s}) for s in (1, 2, 3)])
IDS = [f"{s}-{p}-{'-'.join(f'{k}{v}' for k, v in c.items())}" for s, p, c in CONFIGS]
K = 12


@pytest.fixture(scope="module")
def systems(meshmod, orc):
    m = meshmod.hex_mesh(9, 7, 6)
    a = orc.Addr(m.nCells, m.lower, m.upper)
    p = meshmod.pressure_laplacian(m)
    u = meshmod.momentum_matrix(m)
    sym = orc.Matrix(a, p["diag"], p["upper"])
    asym = orc.Matrix(a, u["diag"], u["upper"], u["lower"])
    b = meshmod.cell_field_global(m, 42)
    psi0 = 0.1 * meshmod.cell_field_global(m, 7)
    return a, sym, asym, b, psi0


def _matrix(systems, solver):
    return systems[1] if solver in ("PCG", "smoothSolver") else systems[2]


@pytest.mark.parametrize("solver,pre,ctl", CONFIGS, ids=IDS)
def test_hook_fed_its_own_sums_changes_nothing(orc, systems, solver, pre, ctl):
    om, b, psi0 = _matrix(systems, solver), systems[3], systems[4]
    ref_psi, ref_perf, ref_hist = om.solve(solver, pre, psi0, b, tolerance=0, maxIter=K, **ctl)
    run = kl.OracleRun(orc, om, solver, pre, psi0, b, staged_ainv=False, tolerance=0, maxIter=K, **ctl)
    rep = kl.Report()
    rep.bits(run.psi, ref_psi, "psi")
    rep.bits(run.hist, ref_hist, "history")
    for f in ("nIterations", "converged", "singular", "initialResidual", "finalResidual", "normFactor"):
        rep.equal(getattr(run.perf, f), getattr(ref_perf, f), f)
    assert run.used, "the hook was never called"
    rep.check()


def _standin(orc, om, solver, pre, psi0, b, maxIter, nudge=None, drop=None, **ctl):
    """the stand-in device: device AINV association, every global sum in numpy's pairwise order.  nudge = (site, it,
    row): the second vector of that product (PCG's p at wApA) is moved one ulp up at that row before it is used;
    drop = (site, it): that sum leaves out its first term"""
    sums = {}

    def fn(site, it, op, x, y, own):
        if nudge and (site, it) == nudge[:2]:
            y[nudge[2]] = np.nextafter(y[nudge[2]], np.inf)
        t = kl.terms_of(op, x, y)
        if drop and (site, it) == drop:
            t = t[1:]
        sums[(site, it)] = float(np.sum(t))
        return sums[(site, it)]

    with orc.ReduceHook(fn, staged_ainv=True):
        psi, perf, hist = om.solve(solver, pre, psi0, b, tolerance=0, maxIter=maxIter, **ctl)
    return psi, perf, hist, sums


def _lockstep(orc, om, solver, pre, psi0, b, k_max, nudge=None, drop=None, **ctl):
    """the comparison the GPU test makes, against the stand-in: per number of bodies k, psi, history and counts bit
    for bit; on the longest run every sum against its bound.  Returns (report, worst ratio)."""
    rep, bound = kl.Report(), kl.Bound()
    n = om.n
    # numpy's pairwise sum: blocks of 8 lanes, then halving; the depth is generous
    depth = lambda nt: 16 + int(np.ceil(np.log2(max(nt, 2))))
    for k in range(1, k_max + 1):
        psi_d, perf_d, hist_d, sums = _standin(orc, om, solver, pre, psi0, b, k - 1, nudge, drop, **ctl)
        checks = []
        on_terms = (lambda s, it, t: checks.append((s, it, t))) if k == k_max else None
        run = kl.OracleRun(orc, om, solver, pre, psi0, b, sums=sums, on_terms=on_terms, staged_ainv=True,
                           tolerance=0, maxIter=k - 1, **ctl)
        tag = f"{solver}/{pre} after iteration {k - 1}"
        rep.equal(run.missing, [], f"{tag}: sums the stand-in did not record")
        rep.bits(run.psi, psi_d, f"{tag}: psi")
        rep.bits(run.hist, hist_d, f"{tag}: history")
        rep.equal(run.perf.nIterations, perf_d.nIterations, f"{tag}: nIterations")
        rep.equal(run.perf.converged, perf_d.converged, f"{tag}: converged")
        for site, it, t in checks:
            bound.check(sums[(site, it)], t, depth(len(t)), f"{solver}/{pre} iteration {it} {site}", rep)
    assert n > 0
    return rep, bound


@pytest.mark.parametrize("solver,pre,ctl", CONFIGS, ids=IDS)
def test_standin_device_in_lockstep(orc, systems, solver, pre, ctl):
    om, b, psi0 = _matrix(systems, solver), systems[3], systems[4]
    rep, bound = _lockstep(orc, om, solver, pre, psi0, b, 8, **ctl)
    print(f"\n[krylov-lockstep-cpu] {solver}/{pre} {ctl}: {bound.checked} sums, worst |s - S| / bound "
          f"{bound.worst:.3g} at {bound.where}")
    assert bound.checked > 0
    rep.check()


def test_one_ulp_in_one_row_is_caught_at_its_iteration(orc, systems):
    """p one ulp off in one row at iteration 3 reaches psi through alpha p at once or, where that rounding absorbs
    it, through the next iterations: the report names the first iteration whose results differ, never an earlier
    one"""
    om, b, psi0 = systems[1], systems[3], systems[4]
    rep, _ = _lockstep(orc, om, "PCG", "DIC", psi0, b, 8, nudge=("wApA", 3, 17))
    assert rep.msgs, "a one-ulp change of p in one row passed"
    first = rep.msgs[0]
    print(f"\n[krylov-lockstep-cpu] p nudged at iteration 3: {first}")
    assert "psi" in first and any(f"after iteration {i}:" in first for i in range(3, 8)), rep.msgs
    assert not any(f"after iteration {i}:" in m for m in rep.msgs for i in range(3)), rep.msgs


def test_dropped_term_fails_the_bound_by_site_and_iteration(orc, systems):
    om, b, psi0 = systems[2], systems[3], systems[4]
    rep, _ = _lockstep(orc, om, "PBiCGStab", "DILU", psi0, b, 5, drop=("tAsA", 2))
    bad = [m for m in rep.msgs if "gamma_" in m]
    assert len(bad) == 1 and "iteration 2 tAsA" in bad[0], rep.msgs
    assert not [m for m in rep.msgs if "psi" in m or "history" in m], rep.msgs
