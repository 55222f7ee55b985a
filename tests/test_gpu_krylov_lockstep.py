"""The device's Krylov solvers and smoothSolver iteration by iteration, bit for bit against the oracle fed the device's
global sums (tests/krylov_lockstep.py).

For every number of iteration bodies k = 1 .. K the device solves with maxIter = k - 1 and an armed trace
(LduMatrix.debug_trace), which records every global sum a scalar step formed and the per-CTA partials it formed it
from.  The oracle then solves the same system with each of its global sums replaced by the device's value for that
site and iteration, and with the device's AINV association (DESIGN.md section 2, exception (i)).  With the order of
the sums taken out, DESIGN.md states the same per-row arithmetic on both sides, so after every k these must be
identical (int64 views): psi, every history entry, nIterations, converged, and the scalars the solve leaves behind
(alpha, beta, omega, rho and the sums they came from).  On the k = K run every device sum is held to the bound of
krylov_lockstep against the exact sum of the oracle's terms, and every per-band partial of a matrix sweep against
the exact sum over that band's rows, so that a wrong or missing row is named by iteration, site and band.

Stated exceptions (DESIGN.md section 2): on the entry stream a row whose terms sum to -0 may come out +0 (psi is
compared with that substitution there); smoothSolver is not run on the cyclic box, whose Jacobi sweep adds the
interface terms in another association (exception (o)).  Only one rank: the peer-memory all-reduce needs several GPUs."""
import importlib

import numpy as np
import pytest

import krylov_lockstep as kl
import polymesh_cases as pc
from test_gpu_engine_streams import engine_env, environ, periodic_problem, random_problem

pytestmark = pytest.mark.gpu

TRACE_CAP = 512


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


class System:
    """one system on the device (one stream, one band size) and in the oracle"""

    def __init__(self, gpu, orc, nCells, lower, upper, diag, up, low=None, patches=(None, None, None), bou=None,
                 centres=None, band=None, fs=None, ctx=None, b=None):
        capi, ctx0, torch = gpu
        self.capi, self.torch = capi, torch
        self.ctx = ctx or ctx0
        self.n = nCells
        with engine_env(band, fs):
            self.addr = capi.LduAddressing(self.ctx, nCells, lower, upper, *patches, cellCentres=centres)
        self.info = self.addr.info()
        self.mat = capi.LduMatrix(self.addr)
        t = lambda a: None if a is None else self.t(a)
        bt = t(bou)  # one tensor for both interface arrays: a matrix with interfaces keeps the face stream so
        self.mat.set(t(diag), t(up), t(low), bt, bt)
        self.mat.debug_trace(TRACE_CAP)
        self.fs = self.info["faceStream"] and low is None
        ps, fc, nr = patches
        if ps is not None:
            self.oa = orc.Addr(nCells, lower, upper, ps, fc, neighbRank=nr)
            self.om = orc.Matrix(self.oa, diag, up, low, bou, bou)
        else:
            self.oa = orc.Addr(nCells, lower, upper)
            self.om = orc.Matrix(self.oa, diag, up, low)
        self.band = self.addr.perm() // self.info["bandRows"]
        self.b = np.random.default_rng(11).standard_normal(nCells) if b is None else b

    def t(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(self.ctx.device)

    def close(self):
        self.mat.close()
        self.addr.close()


def hex_system(gpu, orc, meshmod, dims, kind="P", **kw):
    m = meshmod.hex_mesh(*dims)
    c = meshmod.pressure_laplacian(m) if kind == "P" else meshmod.momentum_matrix(m)
    return System(gpu, orc, m.nCells, m.lower, m.upper, c["diag"], c["upper"], c["lower"] if kind == "U" else None,
                  centres=m.cell_centres(), b=meshmod.cell_field_global(m, 42), **kw)


def poly_system(gpu, orc, kind="P", **kw):
    box = pc.refined_box(10, "random", seed=6)
    if kind == "P":
        _, diag, up = pc.sym_matrix(orc, box)
        low = None
    else:
        _, diag, up, low = pc.asym_matrix(orc, box)
    return System(gpu, orc, box.nCells, box.lower, box.upper, diag, up, low, centres=box.cell_centres(), **kw)


def problem_system(gpu, orc, pb, **kw):
    return System(gpu, orc, pb.nCells, pb.lower, pb.upper, pb.diag, pb.up, patches=(pb.ps, pb.fc, pb.nr), bou=pb.bou,
                  centres=pb.centres, **kw)


def device_solve(sy, solver, pre, psi0, maxIter, **ctl):
    psi = sy.t(psi0)
    perf, hist = sy.mat.solve(solver, pre, psi, sy.t(sy.b), histCap=maxIter + 8, maxIter=maxIter, **ctl)
    return dict(psi=psi.cpu().numpy(), perf=perf, hist=hist, records=sy.mat.debug_get("records"),
                partials=sy.mat.debug_get("partials"), scalars=sy.mat.debug_get("scalars"))


def es_substitute(got, ref):
    """the entry stream's stated exception: +0 where the reference row sums to -0"""
    gb, rb = got.view(np.int64), ref.view(np.int64)
    return np.where((gb == 0) & (rb == np.array(-0.0).view(np.int64)), ref, got)


def lockstep(sy, orc, solver, pre, K, psi0=None, label="", fused=True, tol=0.0, checkEvery=0, **ctl):
    """the comparison of the module docstring for k = 1 .. K (checkEvery: the device's polling interval, 0 its
    default); returns (Report, Bound, the device's k = K solve)"""
    rep, bound = kl.Report(), kl.Bound()
    psi0 = np.zeros(sy.n) if psi0 is None else psi0
    flav = kl.flavour(solver, fused)
    kinds = sy.capi.LduMatrix.STEP_KINDS
    eng = kl.engine_kinds(flav, pre)
    n2 = sy.info["nPadRows"] // 2
    last = None
    for k in range(1, K + 1):
        d = device_solve(sy, solver, pre, psi0, k - 1, tolerance=tol, checkEvery=checkEvery, **ctl)
        tag = f"{label} {solver}/{pre} after iteration {k - 1}"
        if not rep.equal(d["scalars"]["steps"] <= TRACE_CAP, True, f"{tag}: trace overflow"):
            break
        dev = kl.device_sums(flav, d["records"], kinds)
        terms = {}
        on_terms = (lambda s, it, t: terms.__setitem__((s, it), t)) if k == K else None
        run = kl.OracleRun(orc, sy.om, solver, pre, psi0, sy.b, sums={key: v[0] for key, v in dev.items()},
                           on_terms=on_terms, staged_ainv=True, tolerance=tol, maxIter=k - 1, **ctl)
        rep.equal(run.missing, [], f"{tag}: sums the device did not record")
        psi = d["psi"] if sy.fs else es_substitute(d["psi"], run.psi)
        rep.bits(psi, run.psi, f"{tag}: psi")
        rep.bits(d["hist"], run.hist, f"{tag}: history")
        rep.equal(d["perf"].nIterations, run.perf.nIterations, f"{tag}: nIterations")
        rep.equal(d["perf"].converged, run.perf.converged, f"{tag}: converged")
        rep.equal(d["perf"].singular, run.perf.singular, f"{tag}: singular")
        nIt = run.perf.nIterations
        if nIt > 0:
            for f, v in kl.expected_scalars(flav, run.used, nIt - 1).items():
                rep.bits([d["scalars"][f]], [v], f"{tag}: {f}")
        if flav == "pcgFused" and not run.perf.converged:
            rep.equal(int(d["scalars"]["bodies"]), nIt, f"{tag}: bodies")
        if k == K:
            last = d
            for (site, it), t in terms.items():
                if (site, it) not in dev:
                    continue
                s, i, slot = dev[(site, it)]
                r = d["records"][i]
                nP, nred = int(r[2]), int(r[1])
                where = f"{label} {solver}/{pre} iteration {it} {site}"
                bound.check(s, t, kl.sum_depth(n2, nP), where, rep)
                kind = kinds[int(r[0])]
                if kind in eng and len(t) == sy.n:
                    rep.equal(nP, sy.info["nBands"], f"{where}: partials")
                    part = d["partials"][i][: nP * nred].reshape(nP, nred)[:, slot]
                    order = np.argsort(sy.band, kind="stable")
                    cuts = np.searchsorted(sy.band[order], np.arange(nP + 1))
                    ts = t[order]
                    for bnd in range(nP):
                        bound.check(part[bnd], ts[cuts[bnd]:cuts[bnd + 1]], kl.band_depth(n2, nP),
                                    f"{where} band {bnd}", rep)
    return rep, bound, last


def report(rep, bound, what):
    print(f"\n[krylov-lockstep] {what}: {bound.checked} sums and partials, worst |s - S| / bound {bound.worst:.3g} "
          f"at {bound.where}")
    assert bound.checked > 0
    rep.check()


# ---- the cases -----------------------------------------------------------------------------------------------------
PCG_PRE = ("none", "diagonal", "DIC")
ASYM_PRE = ("none", "diagonal", "DILU")


@pytest.fixture(scope="module")
def hex18(gpu, orc, meshmod):
    out = {}

    def get(kind, fs):
        if (kind, fs) not in out:
            out[(kind, fs)] = hex_system(gpu, orc, meshmod, (18, 14, 10), kind, fs=fs)
        return out[(kind, fs)]

    yield get
    for s in out.values():
        s.close()


@pytest.mark.parametrize("fs", (1, 0), ids=("FS", "ES"))
@pytest.mark.parametrize("fused", (1, 0), ids=("fused", "oplist"))
@pytest.mark.parametrize("pre", PCG_PRE)
def test_pcg_hex18(gpu, orc, hex18, pre, fused, fs):
    sy = hex18("P", fs)
    assert sy.fs == bool(fs)
    with environ(B200LDU_PCG_FUSED=fused):
        rep, bound, _ = lockstep(sy, orc, "PCG", pre, 20, label="hex18x14x10", fused=bool(fused))
    report(rep, bound, f"hex18x14x10 PCG/{pre} fused={fused} fs={fs}")


@pytest.mark.parametrize("quirk", (None, 0, 1), ids=("PBiCG", "PBiCGStab-q0", "PBiCGStab-q1"))
@pytest.mark.parametrize("pre", ASYM_PRE)
def test_asym_hex18(gpu, orc, hex18, pre, quirk):
    sy = hex18("U", None)
    solver, ctl = ("PBiCG", {}) if quirk is None else ("PBiCGStab", {"bicgstabRefQuirk": quirk})
    rep, bound, _ = lockstep(sy, orc, solver, pre, 20, label="hex18x14x10", **ctl)
    report(rep, bound, f"hex18x14x10 {solver}/{pre} {ctl}")


@pytest.mark.parametrize("nSweeps", (1, 2, 3))
def test_smooth_hex18(gpu, orc, hex18, nSweeps):
    sy = hex18("P", None)
    rep, bound, _ = lockstep(sy, orc, "smoothSolver", "GaussSeidel", 12, label="hex18x14x10", nSweeps=nSweeps)
    report(rep, bound, f"hex18x14x10 smoothSolver nSweeps={nSweeps}")


@pytest.mark.parametrize("band", (64, 512, 2048))
def test_multislice_bands(gpu, orc, meshmod, band):
    """hex 40x24x20: bands of one to 32 slices on both streams, the fused and the listed PCG, Jacobi and PBiCGStab"""
    rep, bound = kl.Report(), kl.Bound()
    for fs in (1, 0):
        sy = hex_system(gpu, orc, meshmod, (40, 24, 20), band=band, fs=fs)
        try:
            for fused in (1, 0):
                with environ(B200LDU_PCG_FUSED=fused):
                    r, b, _ = lockstep(sy, orc, "PCG", "DIC", 10, label=f"band {band} fs={fs}", fused=bool(fused))
                _merge(rep, bound, r, b)
            if fs:
                r, b, _ = lockstep(sy, orc, "smoothSolver", "GaussSeidel", 6, label=f"band {band}", nSweeps=2)
                _merge(rep, bound, r, b)
        finally:
            sy.close()
    su = hex_system(gpu, orc, meshmod, (40, 24, 20), "U", band=band)
    try:
        r, b, _ = lockstep(su, orc, "PBiCGStab", "DILU", 8, label=f"band {band}")
        _merge(rep, bound, r, b)
    finally:
        su.close()
    report(rep, bound, f"hex40x24x20 band {band}")


def _merge(rep, bound, r, b):
    rep.msgs += r.msgs
    bound.checked += b.checked
    if b.worst > bound.worst:
        bound.worst, bound.where = b.worst, b.where


def _combined(systems, runs):
    rep, bound = kl.Report(), kl.Bound()
    try:
        for sy, args, kw in runs(systems):
            env = kw.pop("env", {})
            with environ(**env):
                r, b, _ = lockstep(sy, *args, **kw)
            _merge(rep, bound, r, b)
    finally:
        for sy in systems:
            sy.close()
    return rep, bound


def test_random_graph_narrowed_bands(gpu, orc):
    pb = random_problem(orc, 4)
    systems = [problem_system(gpu, orc, pb, band=16384, fs=fs) for fs in (1, 0)]
    assert systems[0].info["bandRows"] < 16384
    rep, bound = _combined(systems, lambda s: [
        (s[0], (orc, "PCG", "DIC", 12), dict(label="random30000 FS")),
        (s[1], (orc, "PCG", "DIC", 12), dict(label="random30000 ES")),
        (s[0], (orc, "PCG", "DIC", 12), dict(label="random30000 FS oplist", fused=False,
                                             env={"B200LDU_PCG_FUSED": 0})),
        (s[0], (orc, "smoothSolver", "GaussSeidel", 6), dict(label="random30000", nSweeps=1))])
    report(rep, bound, "random30000")


def test_polyhedral_box(gpu, orc):
    """split-hex box: unsplit cells with up to 24 faces on one side"""
    systems = [poly_system(gpu, orc, "P", fs=1), poly_system(gpu, orc, "P", fs=0, band=64),
               poly_system(gpu, orc, "U", band=2048)]
    rep, bound = _combined(systems, lambda s: [
        (s[0], (orc, "PCG", "DIC", 12), dict(label="poly FS")),
        (s[1], (orc, "PCG", "DIC", 12), dict(label="poly ES band 64")),
        (s[0], (orc, "smoothSolver", "GaussSeidel", 8), dict(label="poly", nSweeps=3)),
        (s[2], (orc, "PBiCG", "DILU", 12), dict(label="poly U")),
        (s[2], (orc, "PBiCGStab", "DILU", 12), dict(label="poly U", bicgstabRefQuirk=0))])
    report(rep, bound, "split-hex box")


def test_cyclic_box(gpu, orc, meshmod):
    """a cyclic pair: the PCG runs its operation list (the fused form needs a peer-memory halo or none)"""
    pb = periodic_problem(meshmod, orc, (24, 20, 16))
    systems = [problem_system(gpu, orc, pb, fs=fs) for fs in (1, 0)]
    rep, bound = _combined(systems, lambda s: [
        (sy, (orc, "PCG", pre, 12), dict(label=f"cyclic fs={fs}", fused=False))
        for sy, fs in zip(s, (1, 0)) for pre in PCG_PRE])
    report(rep, bound, "cyclic 24x20x16")


def test_hex128_default_bands(gpu, orc, meshmod):
    """the benchmark's regime: 2 M cells at the library's own band size"""
    systems = [hex_system(gpu, orc, meshmod, (128, 128, 128))]
    rep, bound = _combined(systems, lambda s: [
        (s[0], (orc, "PCG", "DIC", 8), dict(label="hex128")),
        (s[0], (orc, "PCG", "DIC", 4), dict(label="hex128 oplist", fused=False, env={"B200LDU_PCG_FUSED": 0}))])
    report(rep, bound, "hex128")


# ---- chunking, graphs, a start value, tolerances, poisoned memory ---------------------------------------------------
def _variants(sy, solver, pre, K, psi0, fused=True, **ctl):
    """the same solve under checkEvery 1 / 5 / 8 with graphs on and off: traces and results identical"""
    rep = kl.Report()
    ref = None
    for every in (8, 1, 5):
        for graph in (1, 0):
            with environ(B200LDU_GRAPH=graph):
                d = device_solve(sy, solver, pre, psi0, K - 1, tolerance=0.0, checkEvery=every, **ctl)
            if ref is None:
                ref = d
                continue
            tag = f"{solver}/{pre} checkEvery={every} graph={graph}"
            for f in ("psi", "hist", "records", "partials"):
                rep.bits(d[f], ref[f], f"{tag}: {f}")
            rep.equal(d["scalars"], ref["scalars"], f"{tag}: scalars")
    return rep


@pytest.mark.parametrize("solver,pre,kind,ctl", [("PCG", "DIC", "P", {}), ("PCG", "diagonal", "P", {}),
                                                 ("PBiCGStab", "DILU", "U", {"bicgstabRefQuirk": 0}),
                                                 ("PBiCG", "DILU", "U", {}),
                                                 ("smoothSolver", "GaussSeidel", "P", {"nSweeps": 2})],
                         ids=("PCG-DIC", "PCG-diagonal", "PBiCGStab-DILU", "PBiCG-DILU", "smooth-2"))
def test_chunks_graphs_and_start_value(gpu, orc, meshmod, hex18, solver, pre, kind, ctl):
    sy = hex18(kind, None)
    psi0 = 0.3 * meshmod.cell_field_global(meshmod.hex_mesh(18, 14, 10), 7)
    rep = _variants(sy, solver, pre, 13, psi0, **ctl)  # device only: the oracle knows no chunks
    for every in (1, 5):
        r, b, _ = lockstep(sy, orc, solver, pre, 13, psi0=psi0, label=f"psi0 checkEvery={every}",
                           checkEvery=every, **ctl)
        rep.msgs += r.msgs
    rep.check()


def _stop_tolerance(sy, solver, pre, at, half=False, **ctl):
    """(tolerance, body) that stops the solve at the first body >= at whose residual (for PBiCGStab with half, its
    residual after the half step, sum|sA| / normFactor) lies below every earlier one: the tolerance is just above it"""
    d = device_solve(sy, solver, pre, np.zeros(sy.n), 40, tolerance=0.0, **ctl)
    kinds = sy.capi.LduMatrix.STEP_KINDS
    dev = kl.device_sums(kl.flavour(solver, True), d["records"], kinds)
    nf = dev[("normFactor", 0)][0] + 1e-20
    for j in range(at, 40):
        r = (dev[("sumMagS", j)][0] if half else dev[("sumMag", j)][0]) / nf
        if np.all(d["hist"][: j + 1] > np.nextafter(r, np.inf)):
            return float(np.nextafter(r, np.inf)), j
    raise AssertionError("no body sets a new minimum residual")


@pytest.mark.parametrize("case", ("PCG-fused-in-chunk", "PCG-oplist", "PBiCGStab-half-step"))
def test_tolerance_stops(gpu, orc, hex18, case):
    if case.startswith("PCG"):
        sy, solver, pre, fused = hex18("P", None), "PCG", "DIC", case == "PCG-fused-in-chunk"
        with environ(B200LDU_PCG_FUSED=int(fused)):
            tol, j = _stop_tolerance(sy, solver, pre, 9)
            rep, bound, d = lockstep(sy, orc, solver, pre, j + 4, label=case, fused=fused, tol=tol, checkEvery=4)
        assert d["perf"].converged and d["perf"].nIterations == j + 1
    else:
        sy = hex18("U", None)
        tol, j = _stop_tolerance(sy, "PBiCGStab", "DILU", 5, half=True)
        rep, bound, d = lockstep(sy, orc, "PBiCGStab", "DILU", j + 3, label=case, tol=tol)
        assert d["perf"].converged and d["perf"].nIterations == j + 1
        kinds = sy.capi.LduMatrix.STEP_KINDS
        assert kinds[int(d["records"][-1][0])] == "sMag"  # it stopped at the half step
    report(rep, bound, case)


def test_poisoned_workspace(gpu, orc, meshmod):
    capi, _, torch = gpu
    with environ(B200LDU_POISON_ALLOC=1):
        ctx = capi.Context(0)
    try:
        systems = [hex_system(gpu, orc, meshmod, (18, 14, 10), "P", ctx=ctx),
                   hex_system(gpu, orc, meshmod, (18, 14, 10), "U", ctx=ctx)]
        rep, bound = _combined(systems, lambda s: [
            (s[0], (orc, "PCG", "DIC", 12), dict(label="poisoned")),
            (s[0], (orc, "smoothSolver", "GaussSeidel", 6), dict(label="poisoned", nSweeps=2)),
            (s[1], (orc, "PBiCGStab", "DILU", 12), dict(label="poisoned"))])
        report(rep, bound, "poisoned workspace")
    finally:
        ctx.close()
