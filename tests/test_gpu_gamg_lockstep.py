"""The device GAMG V-cycle level by level and cycle by cycle, bit for bit against the oracle.

After every solve the test reads back what the device built and ran (b200ldu_gamg_debug_get):
 * every level's coarse addressing (owner, neighbour, face restrict map, flips) against the oracle's;
 * every level's coarse coefficients and restricted interface coefficients against the oracle's coarse-matrix accessor;
 * the coarsest inverse, as uploaded, against tests/gamg_levels.gj_inverse of the oracle's coarsest matrix in the
   device's banded numbering (that restatement equals the library's host code, tests/test_gamg_levels_cpu.py);
 * psi against the oracle's V-cycle given that inverse (orc_gamg_set_coarsest_inverse), which applies it as the
   device's kernel does.  With scaleCorrection 0 and one domain a cycle has no global sum in it, so psi after any
   number of cycles matches bit for bit.
Every comparison is of int64 views (-0.0 != +0.0) and a failure names the first differing level and index.

scaleCorrection 1 adds two global sums per level, whose order on the device differs; psi there is held to a bound
measured on the oracle by running the same solve with the two sums in the other order
(tests/gamg_levels.SCALE_REORDER_BOUND)."""
import importlib

import numpy as np
import pytest

import gamg_levels as gl
import polymesh_cases as pc
from test_gpu_engine_streams import engine_env, environ

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


class Case:
    """one mesh and matrix on both sides: oracle (om, og) and device (addr, mat, gg)"""

    def __init__(self, gpu, orc, meshmod, mesh="hex", dims=(16, 14, 12), kind="P", merge=1, band=None, fs=None,
                 ctx=None):
        capi, ctx0, torch = gpu
        self.capi, self.torch = capi, torch
        self.ctx = ctx or ctx0
        patches, bou, intc, coarsest = (None, None, None), None, None, 10
        if mesh == "hex":
            m = meshmod.hex_mesh(*dims)
            c = meshmod.pressure_laplacian(m) if kind == "P" else meshmod.momentum_matrix(m)
            self.n, lower, upper, centres = m.nCells, m.lower, m.upper, m.cell_centres()
            w = meshmod.face_area_pair_weights(m)
            diag, up, low = c["diag"], c["upper"], c["lower"]
            self.oa = orc.Addr(m.nCells, m.lower, m.upper)
            self.b = meshmod.cell_field_global(m, 42)
        elif mesh == "cyclic":  # a box periodic in x: one cyclic patch pair
            from test_oracle_core import _cyclic_case
            m, c, ps, fc, nr, _, _ = _cyclic_case(meshmod, kind)
            self.n, lower, upper, centres = m.nCells, m.lower, m.upper, m.cell_centres()
            w = meshmod.face_area_pair_weights(m)
            diag, up, low, bou, intc = c["diag"], c["upper"], c["lower"], c["bou"], c["int"]
            patches, coarsest = (ps, fc, nr), 4
            self.oa = orc.Addr(m.nCells, m.lower, m.upper, ps, fc, neighbRank=nr)
            self.b = meshmod.cell_field_global(m, 4)
        else:
            box = pc.refined_box(dims, "random", seed=6)
            if kind == "P":
                self.oa, diag, up = pc.sym_matrix(orc, box)
                low = None
            else:
                self.oa, diag, up, low = pc.asym_matrix(orc, box)
            self.n, lower, upper, centres, w = box.nCells, box.lower, box.upper, box.cell_centres(), box.magSf()
            self.b = np.random.default_rng(11).standard_normal(box.nCells)
        self.patches = patches
        self.om = orc.Matrix(self.oa, diag, up, low, bou, intc)
        self.og = orc.Gamg(self.oa, w, coarsest, mergeLevels=merge)
        with engine_env(band, fs):  # the coarse levels' layouts follow the finest level's
            self.addr = capi.LduAddressing(self.ctx, self.n, lower, upper, *patches, cellCentres=centres)
            self.mat = capi.LduMatrix(self.addr)
            self.gg = capi.GamgAgglomeration(self.addr, w, coarsest, mergeLevels=merge)
        self.set(diag, up, low, bou, intc)

    def t(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(self.ctx.device)

    def set(self, diag, up, low, bou=None, intc=None, orc=None):
        t = lambda a: None if a is None else self.t(a)
        self.mat.set(t(diag), t(up), t(low), t(bou), t(intc))
        if orc is not None:
            self.om = orc.Matrix(self.oa, diag, up, low, bou, intc)

    def solve(self, **ctl):
        psi = self.t(np.zeros(self.n))
        perf, hist = self.mat.solve("GAMG", "GaussSeidel", psi, self.t(self.b), gamg=self.gg, histCap=256, **ctl)
        return psi.cpu().numpy(), perf, hist

    def close(self):
        for h in (self.gg, self.mat, self.addr):
            h.close()


def level_mismatches(case, coefficients=True, addressing=True):
    """every difference between the device's levels and the oracle's, level by level (empty: identical)"""
    gg, og, om = case.gg, case.og, case.om
    msgs = []
    assert gg.nLevels == og.nLevels
    for lev in range(gg.nLevels):
        la = og.level_addr(lev)
        if addressing:
            got = gg.level_addressing(lev)
            for name, ref in (("owner", la.lower()), ("neighbour", la.upper()),
                              ("faceRestrict", og.face_restrict_addr(lev)), ("faceFlip", og.face_flip(lev))):
                d = gl.first_difference(got[name], np.asarray(ref, np.int32), exact_int=True)
                if d:
                    msgs.append(f"level {lev} {name} (face): {d}")
        if coefficients:
            cm = og.coarse_matrix(om, lev)
            for name, unit in (("diag", "cell"), ("upper", "face"), ("lower", "face"), ("bou", "patch face"),
                               ("int", "patch face")):
                got = gg.debug_get(lev, name)
                ref = cm[name]
                if ref is None:
                    if got.size:
                        msgs.append(f"level {lev} {name}: the device has one, the symmetric oracle none")
                    continue
                d = gl.first_difference(got, ref)
                if d:
                    msgs.append(f"level {lev} {name} ({unit}): {d}")
    return msgs


def coarsest_reference(case):
    """(device inverse rows, gj_inverse of the oracle's coarsest matrix in the device's banded numbering, perm)"""
    gg, og = case.gg, case.og
    lev = gg.nLevels - 1
    perm = gg.debug_get(lev, "perm")
    n = og.ncells(lev)
    assert np.array_equal(np.sort(perm), np.arange(n)), "coarsest banded rows are not 0..n-1"
    cm, la = og.coarse_matrix(case.om, lev), og.level_addr(lev)
    A = gl.banded_matrix(la.lower(), la.upper(), cm["diag"], cm["upper"], cm["lower"], perm)
    inv, N, off = gg.coarsest_inverse()
    assert (N, off) == (n, 0)
    ref, _ = gl.gj_inverse(A)
    return inv, ref, perm


def check_all(case, psi, perf, ctl):
    """levels, coarsest inverse and psi of the solve just run (from zero, controls ctl) against the oracle"""
    msgs = level_mismatches(case)
    inv, ref, perm = coarsest_reference(case)
    d = gl.first_difference(inv, ref)
    if d:
        msgs.append(f"coarsest inverse (row-major banded): {d}")
    case.og.set_coarsest_inverse(inv, perm)
    psi_ref, pr, _ = case.og.solve(case.om, "GaussSeidel", np.zeros(case.n), case.b,
                                   **oracle_ctl(ctl, tolerance=0.0, relTol=0.0, maxIter=perf.nIterations, minIter=0))
    case.og.set_coarsest_inverse(None)
    assert pr.nIterations == perf.nIterations
    d = gl.first_difference(psi, psi_ref)
    if d:
        msgs.append(f"psi after {perf.nIterations} cycles (cell): {d}")
    assert not msgs, "\n".join(msgs[:12])


BASE = dict(tolerance=0.0, relTol=0.0, scaleCorrection=0)


def oracle_ctl(ctl, **kw):
    """the controls without the device's own (checkEvery: cycles between convergence checks)"""
    return {k: v for k, v in dict(ctl, **kw).items() if k != "checkEvery"}


@pytest.mark.parametrize("kind", ["P", "U"])
@pytest.mark.parametrize("dims", [(16, 14, 12), (9, 9, 9)])
@pytest.mark.parametrize("merge", [1, 2, 3])
def test_levels_and_cycles(gpu, orc, meshmod, kind, dims, merge):
    case = Case(gpu, orc, meshmod, dims=dims, kind=kind, merge=merge)
    try:
        for maxIter in (1, 2, 7, 8, 9, 17):
            ctl = dict(BASE, maxIter=maxIter)
            psi, perf, _ = case.solve(**ctl)
            assert perf.nIterations == maxIter
            check_all(case, psi, perf, ctl)
    finally:
        case.close()


SWEEPS = [dict(nPreSweeps=1), dict(nPreSweeps=2, preSweepsLevelMultiplier=1, maxPreSweeps=3),
          dict(nPostSweeps=1, postSweepsLevelMultiplier=1, maxPostSweeps=3), dict(nFinestSweeps=0),
          dict(nFinestSweeps=1), dict(nFinestSweeps=3), dict(omega=0.8, nPreSweeps=1),
          dict(interpolateCorrection=1), dict(interpolateCorrection=1, nPreSweeps=1, nFinestSweeps=3)]


@pytest.mark.parametrize("kind", ["P", "U"])
@pytest.mark.parametrize("kw", SWEEPS, ids=lambda kw: "-".join(f"{k}{v}" for k, v in kw.items()))
def test_sweep_controls(gpu, orc, meshmod, kind, kw):
    case = Case(gpu, orc, meshmod, kind=kind)
    try:
        for maxIter in (1, 7, 9):
            ctl = dict(BASE, maxIter=maxIter, **kw)
            psi, perf, _ = case.solve(**ctl)
            check_all(case, psi, perf, ctl)
    finally:
        case.close()


@pytest.mark.parametrize("graph", [None, "0"])
@pytest.mark.parametrize("checkEvery", [1, 3, 8])
@pytest.mark.parametrize("nFinest", [1, 2])
def test_check_every_and_graph(gpu, orc, meshmod, graph, checkEvery, nFinest):
    case = Case(gpu, orc, meshmod, kind="P")
    try:
        with environ(B200LDU_GRAPH=graph):
            for maxIter in (1, 2, 7, 8, 9, 17):
                ctl = dict(BASE, maxIter=maxIter, checkEvery=checkEvery, nFinestSweeps=nFinest)
                psi, perf, _ = case.solve(**ctl)
                assert perf.nIterations == maxIter
                check_all(case, psi, perf, ctl)
    finally:
        case.close()


@pytest.mark.parametrize("graph", [None, "0"])
@pytest.mark.parametrize("nFinest", [1, 3])
def test_tolerance_stops_inside_a_chunk(gpu, orc, meshmod, graph, nFinest):
    """A tolerance met after cycle 5 of a chunk of 8, with an odd number of finest sweeps per cycle (psi changes buffer
    every cycle): the device reports 5 cycles and psi is the oracle's after exactly 5."""
    case = Case(gpu, orc, meshmod, kind="P")
    try:
        ctl = dict(BASE, maxIter=40, checkEvery=8, nFinestSweeps=nFinest)
        _, _, href = case.og.solve(case.om, "GaussSeidel", np.zeros(case.n), case.b, **oracle_ctl(ctl))
        k = 5
        assert href[k] < href[k - 1]
        tol = float(np.sqrt(href[k] * href[k - 1]))
        with environ(B200LDU_GRAPH=graph):
            psi, perf, _ = case.solve(**dict(ctl, tolerance=tol))
        assert perf.converged and perf.nIterations == k
        check_all(case, psi, perf, ctl)
    finally:
        case.close()


@pytest.mark.parametrize("kind", ["P", "U"])
@pytest.mark.parametrize("band,fs", [(64, None), (2048, None), (None, 0), (None, 1)])
def test_split_hex_box(gpu, orc, meshmod, kind, band, fs):
    case = Case(gpu, orc, meshmod, mesh="box", dims=10, kind=kind, band=band, fs=fs)
    try:
        for maxIter in (1, 8, 9):
            ctl = dict(BASE, maxIter=maxIter, nFinestSweeps=1)
            psi, perf, _ = case.solve(**ctl)
            check_all(case, psi, perf, ctl)
    finally:
        case.close()


@pytest.mark.parametrize("kind", ["P", "U"])
def test_second_set_of_a_different_matrix(gpu, orc, meshmod, kind):
    """The same handles, a second matrix: the coarse matrices and the inverse read back are the new ones."""
    case = Case(gpu, orc, meshmod, kind=kind)
    try:
        ctl = dict(BASE, maxIter=3)
        psi, perf, _ = case.solve(**ctl)
        check_all(case, psi, perf, ctl)
        old = [case.gg.debug_get(lev, "diag").copy() for lev in range(case.gg.nLevels)]
        m = meshmod.hex_mesh(16, 14, 12)
        c = meshmod.pressure_laplacian(m, seed=99) if kind == "P" else meshmod.momentum_matrix(m, nu=0.003, Co=0.9)
        case.set(c["diag"], c["upper"], c["lower"], orc=orc)
        psi, perf, _ = case.solve(**ctl)
        check_all(case, psi, perf, ctl)
        assert not any(np.array_equal(old[lev], case.gg.debug_get(lev, "diag")) for lev in range(case.gg.nLevels))
    finally:
        case.close()


@pytest.mark.parametrize("kind", ["P", "U"])
def test_cyclic_pair(gpu, orc, meshmod, kind):
    """A box periodic in x (cyclic patch pair): coarse coefficients and restricted interface coefficients bit for bit on
    every level, and the coarsest inverse bit for bit against gj_inverse of the coarsest matrix with every interface
    coefficient at the partner cell's column.  psi is not compared: Jacobi adds the interface terms after the face
    terms (DESIGN.md section 2, exception (o))."""
    case = Case(gpu, orc, meshmod, mesh="cyclic", kind=kind)
    nr = case.patches[2]
    try:
        case.solve(**dict(BASE, maxIter=3))
        msgs = level_mismatches(case)
        lev = case.gg.nLevels - 1
        assert case.og.npatchfaces(lev) > 0
        perm = case.gg.debug_get(lev, "perm")
        cm, la = case.og.coarse_matrix(case.om, lev), case.og.level_addr(lev)
        cps, cfc = la.patch_start(), la.face_cells()
        # the partner of coarse face i of patch p is face i of the partner patch (both sides enumerate the same pairs)
        partner = np.concatenate([cfc[cps[-nr[p] - 1]:cps[-nr[p]]] for p in range(len(nr))])
        A = gl.banded_matrix(la.lower(), la.upper(), cm["diag"], cm["upper"], cm["lower"], perm)
        A = gl.couple(A, cps, cfc, cm["bou"], partner, perm)
        d = gl.first_difference(case.gg.coarsest_inverse()[0], gl.gj_inverse(A)[0])
        if d:
            msgs.append(f"coarsest inverse: {d}")
        assert not msgs, "\n".join(msgs[:12])
    finally:
        case.close()


def test_large_hierarchy(gpu, orc, meshmod):
    """64^3: at least ten levels; coefficients on every level and the coarsest inverse (psi is covered above)"""
    case = Case(gpu, orc, meshmod, dims=(64, 64, 64), kind="P")
    try:
        assert case.gg.nLevels >= 10
        case.solve(**dict(BASE, maxIter=1))
        msgs = level_mismatches(case, addressing=False)
        inv, ref, _ = coarsest_reference(case)
        d = gl.first_difference(inv, ref)
        if d:
            msgs.append(f"coarsest inverse: {d}")
        assert not msgs, "\n".join(msgs[:12])
    finally:
        case.close()


def test_read_back_rules(gpu, orc, meshmod):
    """Coefficients and the inverse exist only after a solve; reading changes nothing a later solve sees."""
    capi = gpu[0]
    case = Case(gpu, orc, meshmod, dims=(9, 9, 9), kind="U")
    try:
        top = case.gg.nLevels - 1
        for name in ("diag", "upper", "lower", "bou", "int", "inv", "invDims"):
            with pytest.raises(capi.B200LduError):
                case.gg.debug_get(top, name)
        assert case.gg.debug_get(0, "owner").size == case.og.nfaces(0)  # addressing needs no solve
        ctl = dict(BASE, maxIter=4)
        psi1, _, _ = case.solve(**ctl)
        for lev in range(case.gg.nLevels):
            case.gg.level_state(lev)
        case.gg.coarsest_inverse()
        with pytest.raises(capi.B200LduError):
            case.gg.debug_get(0, "inv")  # coarsest level only
        psi2, _, _ = case.solve(**ctl)
        assert gl.first_difference(psi1, psi2) is None
    finally:
        case.close()


def test_poisoned_workspace(gpu, orc, meshmod, monkeypatch):
    """B200LDU_POISON_ALLOC=1: every new device block starts NaN; every value read back is finite and still the oracle's."""
    capi = gpu[0]
    monkeypatch.setenv("B200LDU_POISON_ALLOC", "1")
    ctx = capi.Context(0)
    try:
        for kind in ("P", "U"):
            case = Case(gpu, orc, meshmod, dims=(9, 9, 9), kind=kind, ctx=ctx)
            try:
                ctl = dict(BASE, maxIter=7, nFinestSweeps=1, nPreSweeps=1)
                psi, perf, _ = case.solve(**ctl)
                for lev in range(case.gg.nLevels):
                    st = case.gg.level_state(lev)
                    for k, v in st.items():
                        assert v is None or np.all(np.isfinite(v)), (lev, k)
                inv = case.gg.coarsest_inverse()[0]
                assert np.all(np.isfinite(inv)) and np.all(np.isfinite(psi))
                check_all(case, psi, perf, ctl)
            finally:
                case.close()
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", ["P", "U"])
def test_scale_correction(gpu, orc, meshmod, kind):
    case = Case(gpu, orc, meshmod, kind=kind)
    try:
        for kw in gl.SCALE_CTL:
            ctl = dict(tolerance=0.0, relTol=0.0, scaleCorrection=1, **kw)
            psi, perf, _ = case.solve(**ctl)
            assert not level_mismatches(case)
            inv, ref, perm = coarsest_reference(case)
            assert gl.first_difference(inv, ref) is None
            case.og.set_coarsest_inverse(inv, perm)
            psi_ref, pr, _ = case.og.solve(case.om, "GaussSeidel", np.zeros(case.n), case.b, **ctl)
            case.og.set_coarsest_inverse(None)
            assert pr.nIterations == perf.nIterations
            assert gl.rel_diff(psi, psi_ref) <= gl.SCALE_REORDER_BOUND, (kw, gl.rel_diff(psi, psi_ref))
    finally:
        case.close()
