"""No device result may depend on memory nobody wrote.

Every case runs on two contexts: one created with B200LDU_POISON_ALLOC=1, whose handles fill every new floating-point block with
NaNs, and one without.  The two must agree bit for bit, iteration counts and residual histories included, and each agrees with the
oracle to the contract of the existing test of that operation (bit for bit for the matrix operations, face sums, fvMatrix glue,
MULES and field operators; tests/test_gpu_parity.py's contract for solves).

Caller buffers are guarded (`call`): every device array an entry point sees sits in the middle of n + 2G doubles.  Input guards
hold a NaN with payload A, outputs start as NaNs with payload B.  After the call every guard is bit-unchanged (no write past an
end), no payload-B word is left in an output's written range (every element written), nothing outside that range changed, inputs
are unchanged, and the results equal those of the same call on zero-filled buffers (no element past an end was read into a
result).  The shapes are the ragged and degenerate meshes of tests/hygiene_cases.py."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import hygiene_cases as hc
import polymesh_cases as pc
from oracle import fvm_oracle as fo
from test_gpu_engine_streams import environ

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POISON = "B200LDU_POISON_ALLOC"
G = 32                                   # guard doubles on each side: keeps the middle view 256-byte aligned
PAY_A = np.int64(0x7FF80000000A0A0A)     # quiet NaN of the guards
PAY_B = np.int64(0x7FF80000000B0B0B)     # quiet NaN of an output's elements before the call
BANDS = [None, 64]


def dry():
    return os.environ.get("B200LDU_DRYRUN_ORACLE") == "1"


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


# ---- guarded caller buffers ----------------------------------------------------------------------------------------------
def _buffer(torch, dev, n, data, guard, fill):
    host = np.zeros(n + 2 * G)
    if guard:
        host.view(np.int64)[:] = PAY_A
        host.view(np.int64)[G:G + n] = fill
    if data is not None:
        host[G:G + n] = np.asarray(data, np.float64).ravel()
    return torch.from_numpy(host).to(dev)


def call(torch, dev, fn, ins=(), outs=(), inouts=()):
    """fn(views) on guarded buffers, then on zero-padded ones.  ins / inouts: {name: array}; outs: {name: n or (n, lo, hi)} with
    the written range [lo, hi) (default the whole output).  Returns {name: written part of the output or in-out array}."""
    ins, outs, inouts = dict(ins), dict(outs), dict(inouts)
    spec = {k: (len(np.ravel(v)), np.ravel(v), "in", 0, len(np.ravel(v))) for k, v in ins.items()}
    spec.update({k: (len(np.ravel(v)), np.ravel(v), "inout", 0, len(np.ravel(v))) for k, v in inouts.items()})
    for k, v in outs.items():
        n, lo, hi = (v, 0, v) if np.isscalar(v) else v
        spec[k] = (n, None, "out", lo, hi)
    runs = []
    for guard in (True, False):
        bufs = {k: _buffer(torch, dev, n, data, guard, PAY_A if kind == "in" else PAY_B) for k, (n, data, kind, _, _) in spec.items()}
        fn({k: b[G:G + spec[k][0]] for k, b in bufs.items()})
        got = {k: b.cpu().numpy() for k, b in bufs.items()}
        if guard:
            for k, (n, data, kind, lo, hi) in spec.items():
                w = bits(got[k])
                assert (w[:G] == PAY_A).all() and (w[G + n:] == PAY_A).all(), f"{k}: a guard was overwritten"
                mid = w[G:G + n]
                if kind == "in":
                    assert np.array_equal(mid, bits(data)), f"{k}: an input was written"
                elif kind == "out":
                    bad = np.nonzero(mid[lo:hi] == PAY_B)[0]
                    assert not len(bad), f"{k}: {len(bad)} of {hi - lo} elements never written, first {(bad[:4] + lo).tolist()}"
                    assert (mid[:lo] == PAY_B).all() and (mid[hi:] == PAY_B).all(), f"{k}: written outside [{lo}, {hi})"
        runs.append({k: got[k][G:G + n][lo:hi] for k, (n, _, kind, lo, hi) in spec.items() if kind != "in"})
    for k in runs[0]:
        assert np.array_equal(bits(runs[0][k]), bits(runs[1][k])), f"{k}: guarded and zero-padded buffers give different results"
    return runs[0]


def same(a, b, what=""):
    """two results of the two contexts: nested dicts / tuples of arrays and numbers, bit for bit"""
    if isinstance(a, dict):
        assert sorted(map(str, a)) == sorted(map(str, b)), what
        for k in a:
            same(a[k], b[k], f"{what}/{k}")
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            same(x, y, f"{what}[{i}]")
    elif a is None or isinstance(a, str):
        assert a == b, what
    else:
        x, y = np.asarray(a, np.float64), np.asarray(b, np.float64)
        assert x.shape == y.shape and np.array_equal(bits(x), bits(y)), f"poisoned and clean contexts differ: {what}"


# ---- contexts ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctxs = {}
    for poison in (True, False):
        with environ(**{POISON: "1" if poison else None}):
            ctxs[poison] = capi.Context(0)
    yield capi, ctxs, torch
    for c in ctxs.values():
        c.close()


class Dev:
    """one shape's addressing and matrix on one context"""

    def __init__(self, capi, ctx, torch, box, coeffs, band=None, fs=None):
        self.capi, self.ctx, self.torch, self.box = capi, ctx, torch, box
        self.dev, self.L, self.dp = ctx.device, capi.lib(), capi._dp
        with environ(B200LDU_BAND_ROWS=band, B200LDU_FACE_STREAM=fs):
            self.addr = capi.mesh_to_device(ctx, box)
        capi.fv_boundary_set(self.addr, box.bFaceCells)
        self.mat = capi.LduMatrix(self.addr)
        if coeffs is not None:
            self.set(coeffs)

    def t(self, a):
        return self.torch.from_numpy(np.array(a, dtype=np.float64).ravel()).to(self.dev)

    def set(self, coeffs):
        self.keep = [None if c is None else self.t(c) for c in coeffs]
        self.mat.set(*self.keep)

    def call(self, fn, ins=(), outs=(), inouts=()):
        return call(self.torch, self.dev, fn, ins, outs, inouts)

    def close(self):
        self.mat.close()
        self.addr.close()


def both(gpu, run):
    """run(capi, ctx, torch) on the poisoned and the clean context; the results agree bit for bit.  Returns the clean one."""
    capi, ctxs, torch = gpu
    res = {p: run(capi, ctxs[p], torch) for p in (True, False)}
    same(res[True], res[False])
    return res[False]


# ---- a. matrix operations, preconditioners, smoothers and the banded views ----------------------------------------------
def _ops(capi, ctx, torch, box, coeffs, band, fs, x, b):
    D = Dev(capi, ctx, torch, box, coeffs, band, fs)
    L, dp, h = D.L, D.dp, D.mat.h
    n, nF, vl = box.nCells, box.nFaces, D.addr.vec_len
    r = {}
    for name, fn in (("Amul", L.b200ldu_amul), ("Tmul", L.b200ldu_tmul), ("H", L.b200ldu_H)):
        r[name] = D.call(lambda v, fn=fn: capi.check(fn(h, dp(v["x"]), dp(v["y"]))), {"x": x}, {"y": n})["y"]
    if nF:              # without faces faceH is an error, as lduMatrix::faceH is
        r["faceH"] = D.call(lambda v: capi.check(L.b200ldu_faceH(h, dp(v["x"]), dp(v["y"]))), {"x": x}, {"y": nF})["y"]
    else:
        with pytest.raises(capi.B200LduError):
            D.call(lambda v: capi.check(L.b200ldu_faceH(h, dp(v["x"]), dp(v["y"]))), {"x": x}, {"y": nF})
    r["sumA"] = D.call(lambda v: capi.check(L.b200ldu_sumA(h, dp(v["y"]))), (), {"y": n})["y"]
    r["H1"] = D.call(lambda v: capi.check(L.b200ldu_H1(h, dp(v["y"]))), (), {"y": n})["y"]
    r["residual"] = D.call(lambda v: capi.check(L.b200ldu_residual(h, dp(v["x"]), dp(v["b"]), dp(v["y"]))), {"x": x, "b": b},
                           {"y": n})["y"]
    for pre in ("none", "diagonal", "DIC", "DILU"):
        for T in (0, 1):
            r[f"{pre}{T}"] = D.call(lambda v: capi.check(L.b200ldu_precondition(h, pre.encode(), T, dp(v["x"]), dp(v["y"]))),
                                    {"x": x}, {"y": n})["y"]
    for sm in ("Jacobi", "GaussSeidel"):
        for ns in (1, 2):
            r[f"{sm}{ns}"] = D.call(lambda v: capi.check(L.b200ldu_smooth(h, sm.encode(), 0.9, dp(v["psi"]), dp(v["b"]), ns)),
                                    {"b": b}, (), {"psi": x})["psi"]
    nPad = D.addr.info()["nPadRows"]
    # to_banded writes the real and padding rows; the receive tail is the halo exchange's
    xb = D.call(lambda v: capi.check(L.b200ldu_to_banded(D.addr.h, dp(v["x"]), dp(v["xb"]))), {"x": x}, {"xb": (vl, 0, nPad)})["xb"]
    r["to_banded"] = xb
    r["from_banded"] = D.call(lambda v: capi.check(L.b200ldu_from_banded(D.addr.h, dp(v["xb"]), dp(v["x"]))),
                              {"xb": np.concatenate([xb, np.zeros(vl - nPad)])}, {"x": n})["x"]
    # amul_banded exchanges the halo into the receive tail [nPad, vec_len) of its input first: an in-out array whose rows stay
    yb = D.call(lambda v: capi.check(L.b200ldu_amul_banded(h, dp(v["xb"]), dp(v["yb"]))), (), {"yb": (vl, 0, nPad)},
                {"xb": np.concatenate([xb, np.zeros(vl - nPad)])})
    assert np.array_equal(bits(yb["xb"][:nPad]), bits(xb))
    r["amul_banded"] = yb["yb"]
    r["perm"] = D.addr.perm().astype(np.float64)
    r["nPad"] = float(nPad)
    D.close()
    return r


@pytest.mark.parametrize("fs", [None, 0, 1])
@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("band", BANDS)
@pytest.mark.parametrize("name", hc.NAMES)
def test_matrix_operations(gpu, orc, name, band, symmetric, fs):
    if fs is not None and not symmetric:
        pytest.skip("the face stream serves symmetric matrices only")
    box = hc.build(name)
    coeffs = hc.coefficients(box, symmetric, 3)
    _, om = hc.oracle_matrix(orc, box, coeffs)
    rng = np.random.default_rng(4)
    x, b = rng.uniform(-1, 1, box.nCells), rng.uniform(-1, 1, box.nCells)
    r = both(gpu, lambda capi, ctx, torch: _ops(capi, ctx, torch, box, coeffs, band, fs, x, b))
    coupled = coeffs[3] is not None
    for k, want in (("Amul", om.amul(x)), ("Tmul", om.tmul(x)), ("H", om.H(x)), ("sumA", om.sumA()), ("H1", om.H1()),
                    ("residual", om.residual(x, b)), ("faceH", om.faceH(x) if box.nFaces else None)):
        assert want is None or np.array_equal(r[k], want), k
    for pre in ("none", "diagonal", "DIC", "DILU"):
        for T in (0, 1):
            want = om.precondition(pre, x, bool(T))
            if pre in ("DIC", "DILU"):     # the AINV staging: one rounding per term apart (tests/test_gpu_parity.py)
                np.testing.assert_allclose(r[f"{pre}{T}"], want, rtol=1e-13, atol=1e-13 * np.abs(want).max(initial=0.0))
            else:
                assert np.array_equal(r[f"{pre}{T}"], want), (pre, T)
    for sm in ("Jacobi", "GaussSeidel"):
        for ns in (1, 2):
            want = om.jacobi(x, b, ns)
            if coupled:                    # interface terms after the face terms (DESIGN.md section 2, exception (o))
                np.testing.assert_allclose(r[f"{sm}{ns}"], want, rtol=1e-13, atol=1e-14)
            else:
                assert np.array_equal(r[f"{sm}{ns}"], want), (sm, ns)
    perm, nPad = r["perm"].astype(int), int(r["nPad"])
    want_b = np.zeros(nPad)
    want_b[perm] = x
    assert np.array_equal(bits(r["to_banded"]), bits(want_b)), "to_banded: real rows in place, padding rows +0"
    assert np.array_equal(r["from_banded"], x)
    if not coupled:
        assert np.array_equal(r["amul_banded"][perm], om.amul(x))
        assert np.array_equal(r["amul_banded"][np.setdiff1d(np.arange(nPad), perm)], np.zeros(nPad - box.nCells))


# ---- b. solvers ----------------------------------------------------------------------------------------------------------
def _cmp_hist(h, href):
    """tests/test_gpu_parity.py's contract on meshes this small (its cyclic case): the global sums' order shows within a few
    iterations, so rel 1e-8 over the first 10 and 1e-3 over the first 30, each with a floor"""
    for first, rtol in ((10, 1e-8), (30, 1e-3)):
        k = min(first, len(h), len(href))
        np.testing.assert_allclose(np.asarray(h[:k]), np.asarray(href[:k]), rtol=rtol, atol=rtol * 1e-6)


def _perf(p):
    return (p.initialResidual, p.finalResidual, p.normFactor, p.nIterations, p.converged, p.singular)


def _solve(D, solver, pre, x0, b, gamg=None, histCap=256, env=None, **ctl):
    capi, L, dp, h = D.capi, D.L, D.dp, D.mat.h
    c = capi.controls(**ctl)
    perf = capi.Perf()
    hist = np.full(max(histCap, 1), np.nan)
    rc = []

    def fn(v):
        with environ(**(env or {})):
            rc.append(L.b200ldu_solve(h, solver.encode(), pre.encode(), capi.C.byref(c), gamg.h if gamg is not None else None,
                                      dp(v["psi"]), dp(v["b"]), capi.C.byref(perf), hist.ctypes.data_as(capi.vp), histCap))
    psi = D.call(fn, {"b": b}, (), {"psi": x0})["psi"]
    assert rc[0] == rc[1]
    if rc[0] != 0:
        return rc[0], psi, None, None
    return 0, psi, _perf(perf), hist[~np.isnan(hist)]


SYM_SOLVES = [("PCG", "DIC", dict(checkEvery=1), {"B200LDU_PCG_FUSED": "1"}),
              ("PCG", "DIC", dict(checkEvery=8), {"B200LDU_PCG_FUSED": "1"}),
              ("PCG", "diagonal", dict(checkEvery=1), {"B200LDU_PCG_FUSED": "0"}),
              # without a preconditioner the recurrence on the hub amplifies the order of the global sums to 6e-4 by iteration 9
              ("PCG", "diagonal", dict(checkEvery=8), {"B200LDU_PCG_FUSED": "0"}),
              ("ICCG", "", {}, None), ("diagonal", "", {}, None), ("smoothSolver", "GaussSeidel", dict(nSweeps=2), None),
              ("PCG", "DIC", dict(maxIter=0), None)]
ASYM_SOLVES = [("PBiCG", "DILU", {}, None), ("PBiCGStab", "DILU", {}, None), ("BICCG", "", {}, None),
               ("smoothSolver", "Jacobi", dict(nSweeps=1), None), ("PBiCG", "diagonal", dict(maxIter=0), None)]


def _solves(capi, ctx, torch, box, coeffs, band, x0, b, solves, merges):
    D = Dev(capi, ctx, torch, box, coeffs, band)
    r = {}
    for i, (solver, pre, kw, env) in enumerate(solves):
        ctl = dict(dict(tolerance=1e-7, maxIter=300), **kw)
        r[i] = _solve(D, solver, pre, x0, b, env=env, **ctl)[1:]
    solver, pre = solves[0][:2]
    r["zero"] = _solve(D, solver, pre, x0, np.zeros(box.nCells), tolerance=1e-7, maxIter=300)[1:]
    ph, bh = x0.copy(), b.copy()
    perf = D.mat.solve_host(solver, pre, ph, bh, tolerance=1e-7, maxIter=300)
    r["host"] = (ph, _perf(perf))
    fw = np.abs(coeffs[1]) if box.nFaces else np.zeros(0)
    for merge in merges:
        try:
            g = capi.GamgAgglomeration(D.addr, fw, 4, merge)
        except capi.B200LduError as e:
            r[f"gamg{merge}"] = ("create", e.rc)
            continue
        r[f"gamg{merge}"] = (g.nLevels,) + _solve(D, "GAMG", "GaussSeidel", x0, b, gamg=g, tolerance=1e-7, maxIter=100)
        g.close()
    D.close()
    return r


@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("band", BANDS)
@pytest.mark.parametrize("name", hc.NAMES)
def test_solvers(gpu, orc, name, band, symmetric):
    box = hc.build(name)
    coeffs = hc.coefficients(box, symmetric, 5)
    oa, om = hc.oracle_matrix(orc, box, coeffs)
    rng = np.random.default_rng(6)
    x0, b = rng.uniform(-1, 1, box.nCells), rng.uniform(-1, 1, box.nCells)
    solves = SYM_SOLVES if symmetric else ASYM_SOLVES
    r = both(gpu, lambda capi, ctx, torch: _solves(capi, ctx, torch, box, coeffs, band, x0, b, solves, (1, 2)))
    checks = [(i, s, p, dict(dict(tolerance=1e-7, maxIter=300), **kw)) for i, (s, p, kw, _) in enumerate(solves)]
    checks.append(("zero", solves[0][0], solves[0][1], dict(tolerance=1e-7, maxIter=300)))
    for key, solver, pre, ctl in checks:
        ctl = {k: v for k, v in ctl.items() if k != "checkEvery"}
        src = np.zeros(box.nCells) if key == "zero" else b
        psi_ref, pr, href = om.solve(solver, pre, x0, src, **ctl)
        psi, perf, hist = r[key]
        assert perf is not None, (key, solver, pre)
        assert abs(perf[3] - pr.nIterations) <= 1 + pr.nIterations // 10, (key, solver, pre, perf[3], pr.nIterations)
        # maxIter 0 still runs one iteration (the do-while loops of PCG.C, PBiCG.C)
        assert ctl.get("maxIter") == 0 or perf[4] == pr.converged, (key, solver, pre)
        _cmp_hist(hist, href)
        np.testing.assert_allclose(psi, psi_ref, rtol=0, atol=1e-5 * max(1.0, np.abs(psi_ref).max()))
    ph, perf = r["host"]
    psi_ref, pr, _ = om.solve(solves[0][0], solves[0][1], x0, b, tolerance=1e-7, maxIter=300)
    assert abs(perf[3] - pr.nIterations) <= 1 + pr.nIterations // 10
    np.testing.assert_allclose(ph, psi_ref, rtol=0, atol=1e-5 * max(1.0, np.abs(psi_ref).max()))
    fw = np.abs(coeffs[1]) if box.nFaces else np.zeros(0)
    for merge in (1, 2):
        got = r[f"gamg{merge}"]
        if not box.nFaces:      # a matrix without off-diagonal coefficients is solved by the diagonal solver, whatever was asked
            assert got[:2] == (0, 0) and np.array_equal(got[2], b / coeffs[0]), (merge, got[:2])
            continue
        og = orc.Gamg(oa, fw, 4, merge)
        if og.nLevels == 0:
            # no hierarchy: the solve refuses with B200LDU_ENOLEVELS and leaves psi as it was
            assert got[0] == "create" or (got[0] == 0 and got[1] == -8 and np.array_equal(bits(got[2]), bits(x0))), (merge, got[:2])
            continue
        assert got[0] == og.nLevels and got[1] == 0, (merge, got[:2])
        psi_ref, pr, href = og.solve(om, "GaussSeidel", x0, b, tolerance=1e-7, maxIter=100)
        psi, perf, hist = got[2:]
        assert perf[3] == pr.nIterations, (merge, perf[3], pr.nIterations)
        np.testing.assert_allclose(hist[: len(href)], href, rtol=1e-6, atol=1e-15)     # as test_gpu_parity's cyclic GAMG
        np.testing.assert_allclose(psi, psi_ref, rtol=0, atol=1e-5 * max(1.0, np.abs(psi_ref).max()))


# ---- c. finite-volume face sums, limited fluxes, MULES and the fvMatrix glue --------------------------------------------
def _fv(capi, ctx, torch, box, band, data):
    D = Dev(capi, ctx, torch, box, None, band)
    L, dp, A = D.L, D.dp, D.addr.h
    n, nF, nB = box.nCells, box.nFaces, len(box.bFaceCells)
    d = data
    r = {}
    for nc in (1, 3):
        for div, sign in ((1, -1), (0, 1)):
            r[f"si{nc}{div}"] = D.call(lambda v: capi.check(L.b200ldu_fv_surface_integrate(A, nc, dp(v["s"]), dp(v["bs"]), dp(v["V"]),
                                                                                           dp(v["o"]), div, sign)),
                                       {"s": d[f"ssf{nc}"], "bs": d[f"bssf{nc}"], "V": d["V"]}, {"o": n * nc})["o"]
        r[f"gg{nc}"] = D.call(lambda v: capi.check(L.b200ldu_fv_gauss_grad(A, nc, dp(v["Sf"]), dp(v["s"]), dp(v["bSf"]), dp(v["bs"]),
                                                                           dp(v["V"]), dp(v["o"]))),
                              {"Sf": d["Sf"], "s": d[f"ssf{nc}"], "bSf": d["bSf"], "bs": d[f"bssf{nc}"], "V": d["V"]}, {"o": 3 * n * nc})["o"]
        r[f"il{nc}"] = D.call(lambda v: capi.check(L.b200ldu_fv_interpolate_linear(A, nc, dp(v["w"]), dp(v["vf"]), dp(v["o"]))),
                              {"w": d["w"], "vf": d[f"vf{nc}"]}, {"o": nF * nc})["o"]
        r[f"sn{nc}"] = D.call(lambda v: capi.check(L.b200ldu_fv_sngrad(A, nc, dp(v["dc"]), dp(v["vf"]), dp(v["o"]))),
                              {"dc": d["dc"], "vf": d[f"vf{nc}"]}, {"o": nF * nc})["o"]
    r["lap"] = D.call(lambda v: capi.check(L.b200ldu_fv_laplacian_fill(A, dp(v["dc"]), dp(v["g"]), dp(v["u"]), dp(v["d"]))),
                      {"dc": d["dc"], "g": d["g"]}, {"u": nF, "d": n})
    r["conv"] = D.call(lambda v: capi.check(L.b200ldu_fv_convection_fill(A, dp(v["w"]), dp(v["phi"]), dp(v["l"]), dp(v["u"]),
                                                                         dp(v["d"]))),
                       {"w": d["w"], "phi": d["phi"]}, {"l": nF, "u": nF, "d": n})
    r["abd"] = D.call(lambda v: capi.check(L.b200ldu_fv_add_boundary_diag(A, dp(v["ic"]), dp(v["d"]))), {"ic": d["ic"]}, (),
                      {"d": d["d0"]})["d"]
    for scheme, k in (("upwind", 1.0), ("limitedLinear", 0.5), ("vanLeer", 1.0)):
        r[f"lim{scheme}"] = D.call(lambda v: capi.check(L.b200ldu_fv_limiter(A, scheme.encode(), k, dp(v["f"]), dp(v["vf"]), dp(v["gc"]),
                                                                             dp(v["C"]), dp(v["o"]))),
                                   {"f": d["phi"], "vf": d["vf1"], "gc": d["gradc"], "C": d["C"]}, {"o": nF})["o"]
        r[f"lf{scheme}"] = D.call(lambda v: capi.check(L.b200ldu_fv_limited_flux(A, scheme.encode(), k, dp(v["f"]), dp(v["vf"]),
                                                                                 dp(v["gc"]), dp(v["C"]), dp(v["cd"]), -1, 1, dp(v["o"]))),
                                  {"f": d["phi"], "vf": d["vf1"], "gc": d["gradc"], "C": d["C"], "cd": d["w"]}, {"o": nF})["o"]
    r["vof"] = D.call(lambda v: capi.check(L.b200ldu_vof_interface_flux(A, dp(v["w"]), dp(v["g"]), dp(v["Sf"]), dp(v["bSf"]),
                                                                        dp(v["bSn"]), 1e-8, dp(v["phi"]), dp(v["m"]), 0.75,
                                                                        dp(v["n"]), dp(v["nB"]), dp(v["p"]))),
                      {"w": d["w"], "g": d["ga"], "Sf": d["Sf"], "bSf": d["bSf"], "bSn": d["bSn"], "phi": d["phi"], "m": d["magSf"]},
                      {"n": nF, "nB": nB, "p": nF})
    M = d["mules"]
    mins = {k: M[k] for k in ("V", "psi", "psi0", "psiB", "bd", "bdB", "corr", "corrB")}
    r["mules"] = D.call(lambda v: capi.check(L.b200ldu_mules_limiter(A, 3, M["rDeltaT"], None, None, dp(v["psi"]), dp(v["psi0"]),
                                                                     dp(v["psiB"]), dp(v["bd"]), dp(v["bdB"]), dp(v["corr"]),
                                                                     dp(v["corrB"]), None, None, dp(v["V"]), 1.0, 0.0, dp(v["lam"]),
                                                                     dp(v["lamB"]), 0)),
                        mins, (), {"lam": np.ones(nF), "lamB": np.ones(nB)})
    cins = {k: M[k] for k in ("V", "psi", "psiB", "phiB", "corr", "corrB")}
    r["mulesc"] = D.call(lambda v: capi.check(L.b200ldu_mules_limiter_corr(A, 3, M["rDeltaT"], None, dp(v["psi"]), dp(v["psiB"]),
                                                                           dp(v["phiB"]), dp(v["corr"]), dp(v["corrB"]), None, None,
                                                                           dp(v["V"]), 1.0, 0.0, 0.2, dp(v["lam"]), dp(v["lamB"]), 0)),
                         cins, (), {"lam": np.ones(nF), "lamB": np.ones(nB)})
    F = d["fvm"]
    D.set((F["diag"], F["upper"], F["lower"], None, None))
    h = D.mat.h
    r["fvmA"] = D.call(lambda v: capi.check(L.b200ldu_fvm_A(h, 1, dp(v["ic"]), dp(v["V"]), dp(v["o"]))), {"ic": F["ic"], "V": F["V"]},
                       {"o": n})["o"]
    r["fvmH"] = D.call(lambda v: capi.check(L.b200ldu_fvm_H(h, 1, dp(v["psi"]), dp(v["s"]), dp(v["bc"]), None, dp(v["V"]), dp(v["o"]))),
                       {"psi": F["x"], "s": F["source"], "bc": F["bc"], "V": F["V"]}, {"o": n})["o"]
    r["fvmR"] = D.call(lambda v: capi.check(L.b200ldu_fvm_residual(h, dp(v["psi"]), dp(v["s"]), dp(v["ic"]), dp(v["bc"]), None,
                                                                   dp(v["o"]))),
                       {"psi": F["x"], "s": F["source"], "ic": F["ic"], "bc": F["bc"]}, {"o": n})["o"]
    r["fvmF"] = D.call(lambda v: capi.check(L.b200ldu_fvm_flux(h, 1, dp(v["psi"]), dp(v["ic"]), dp(v["bc"]), None, dp(v["f"]),
                                                               dp(v["b"]), dp(v["c"]))),
                       {"psi": F["x"], "ic": F["ic"], "bc": F["bc"]}, {"f": nF, "b": nB, "c": (1, 0, 0)})
    r["relax"] = D.call(lambda v: capi.check(L.b200ldu_fvm_relax(h, 1, 0.7, dp(v["psi"]), dp(v["ic"]), dp(v["d"]), dp(v["s"]))),
                        {"psi": F["x"], "ic": F["ic"]}, (), {"d": F["diag"], "s": F["source"]})
    val = np.array([0.75])
    r["ref"] = D.call(lambda v: capi.check(L.b200ldu_fvm_set_reference(h, n - 1, 1, val.ctypes.data_as(capi.vp), dp(v["d"]),
                                                                       dp(v["s"]))), (), (), {"d": F["diag"], "s": F["source"]})
    D.close()
    return r


def _fv_data(orc, box):
    from oracle import interfoam_oracle as io
    from oracle import mules_oracle as mo
    rng = np.random.default_rng(8)
    n, nF, nB = box.nCells, box.nFaces, len(box.bFaceCells)
    oa = pc.addr(orc, box)
    d = dict(V=box.volumes(), Sf=box.Sf(), bSf=box.bSf, w=box.weights(), dc=box.deltaCoeffs(), C=box.cell_centres(), magSf=box.magSf())
    for nc in (1, 3):
        d[f"ssf{nc}"], d[f"bssf{nc}"], d[f"vf{nc}"] = rng.uniform(-1, 1, (nF, nc)), rng.uniform(-1, 1, (nB, nc)), rng.uniform(-1, 1, (n, nc))
    d["g"] = rng.uniform(0.5, 1.5, nF) * box.magSf()
    d["phi"] = rng.uniform(-1, 1, nF)
    d["phi"][::7] = 0.0
    d["ic"], d["d0"] = rng.uniform(-1, 1, nB), rng.uniform(1, 2, n)
    sf = np.asarray(orc.interpolate_linear(oa, d["w"], d["vf1"].ravel(), 1)).ravel()
    d["gradc"] = np.asarray(orc.gauss_grad(oa, box.Sf().ravel(), sf, box.bFaceCells, box.bSf.ravel(), d["bssf1"].ravel(), d["V"], 1))
    d["ga"] = rng.uniform(-1, 1, (n, 3))
    d["bSn"] = rng.uniform(-1, 1, nB)
    M = pc.mules_case(box, 12)
    M["bd"], M["bdB"] = mo.upwind_flux(box.lower, box.upper, M["phi"], M["phiB"], M["psi"], M["psiB"])
    M["corr"], M["corrB"] = M["phiPsi"] - M["bd"], M["phiPsiB"] - M["bdB"]
    d["mules"] = M
    _, F, _ = pc.fvm_case(orc, box, 1, 3)
    F["x"] = rng.uniform(-1, 1, n)
    d["fvm"] = F
    return oa, d, io, mo


@pytest.mark.parametrize("band", BANDS)
@pytest.mark.parametrize("name", hc.FV_NAMES)
def test_finite_volume(gpu, orc, name, band):
    from test_oracle_fvm import make
    box = hc.build(name)
    oa, d, io, mo = _fv_data(orc, box)
    r = both(gpu, lambda capi, ctx, torch: _fv(capi, ctx, torch, box, band, d))
    bfc, L, U = box.bFaceCells, box.lower, box.upper
    eq = lambda got, want, what: np.testing.assert_array_equal(np.ravel(got), np.ravel(np.asarray(want)), err_msg=what)
    for nc in (1, 3):
        for div, sign in ((1, -1), (0, 1)):
            eq(r[f"si{nc}{div}"], orc.surface_integrate(oa, d[f"ssf{nc}"].ravel(), bfc, d[f"bssf{nc}"].ravel(), d["V"], nc, bool(div), sign),
               f"surface_integrate {nc} {div}")
        eq(r[f"gg{nc}"], orc.gauss_grad(oa, d["Sf"].ravel(), d[f"ssf{nc}"].ravel(), bfc, d["bSf"].ravel(), d[f"bssf{nc}"].ravel(), d["V"], nc),
           f"gauss_grad {nc}")
        eq(r[f"il{nc}"], orc.interpolate_linear(oa, d["w"], d[f"vf{nc}"].ravel(), nc), f"interpolate {nc}")
        eq(r[f"sn{nc}"], orc.sngrad(oa, d["dc"], d[f"vf{nc}"].ravel(), nc), f"sngrad {nc}")
    ru, rd = orc.laplacian_fill(oa, d["dc"], d["g"])
    eq(r["lap"]["u"], ru, "laplacian upper"), eq(r["lap"]["d"], rd, "laplacian diag")
    rl, ru, rd = orc.convection_fill(oa, d["w"], d["phi"])
    eq(r["conv"]["l"], rl, "conv lower"), eq(r["conv"]["u"], ru, "conv upper"), eq(r["conv"]["d"], rd, "conv diag")
    eq(r["abd"], orc.add_boundary_diag(bfc, d["ic"], d["d0"]), "add_boundary_diag")
    for scheme, k in (("upwind", 1.0), ("limitedLinear", 0.5), ("vanLeer", 1.0)):
        eq(r[f"lf{scheme}"], io.limited_flux(scheme, L, U, d["phi"], d["vf1"].ravel(), d["gradc"].reshape(-1, 3), d["C"], d["w"], k, -1, 1),
           f"limited_flux {scheme}")
    w0, w1, w2 = io.interface_flux(L, U, d["w"], d["ga"], d["Sf"], bfc, d["bSf"], d["bSn"], 1e-8, d["phi"], d["magSf"], 0.75)
    eq(r["vof"]["n"], w0, "nHatf"), eq(r["vof"]["nB"], w1, "nHatfB"), eq(r["vof"]["p"], w2, "phir")
    M = d["mules"]
    want, wantB = mo.limiter(box.nCells, L, U, bfc, M["V"], M["rDeltaT"], M["psi"], M["psi0"], M["psiB"], M["bd"], M["bdB"], M["corr"],
                             M["corrB"], 1.0, 0.0, 3)
    eq(r["mules"]["lam"], want, "mules lambda"), eq(r["mules"]["lamB"], wantB, "mules lambdaB")
    want, wantB = mo.limiter(box.nCells, L, U, bfc, M["V"], M["rDeltaT"], M["psi"], M["psi"], M["psiB"], np.zeros(box.nFaces), M["phiB"],
                             M["corr"], M["corrB"], 1.0, 0.0, 3, corr=True, extremaCoeff=0.2)
    eq(r["mulesc"]["lam"], want, "limiterCorr lambda"), eq(r["mulesc"]["lamB"], wantB, "limiterCorr lambdaB")
    F = d["fvm"]
    ofm = make(orc, oa, F, 1, F["x"].reshape(-1, 1))
    eq(r["fvmA"], ofm.A(), "fvm A"), eq(r["fvmH"], ofm.H(), "fvm H"), eq(r["fvmR"], ofm.residual(), "fvm residual")
    oi, ob, _ = ofm.flux()
    eq(r["fvmF"]["f"], oi, "fvm flux"), eq(r["fvmF"]["b"], ob, "fvm boundary flux")
    orl = make(orc, oa, F, 1, F["x"].reshape(-1, 1))
    orl.relax(0.7)
    eq(r["relax"]["d"], orl.diag, "relax diag"), eq(r["relax"]["s"], orl.source, "relax source")
    ors = make(orc, oa, F, 1, F["x"].reshape(-1, 1))
    ors.setReference(box.nCells - 1, [0.75])
    eq(r["ref"]["d"], ors.diag, "setReference diag"), eq(r["ref"]["s"], ors.source, "setReference source")


def _ldu_no_faces(capi, ctx, torch, box, A, B, sf):
    D = Dev(capi, ctx, torch, box, None)
    L, dp, a = D.L, D.dp, D.addr.h
    hasA, hasB = (capi.C.c_int * 3)(1, 1, 1), (capi.C.c_int * 3)(1, 1, 0)
    r = {}
    for sub in (0, 1):
        r[f"aa{sub}"] = D.call(lambda v: capi.check(L.b200ldu_ldu_add_assign(a, sub, dp(v["d"]), dp(v["u"]), dp(v["l"]), hasA, dp(v["od"]),
                                                                             dp(v["ou"]), None, hasB)),
                               {"od": B["diag"], "ou": np.zeros(1)}, (), {"d": A["diag"], "u": np.zeros(1), "l": np.zeros(1)})
    r["scale"] = D.call(lambda v: capi.check(L.b200ldu_ldu_scale(a, dp(v["sf"]), 0.0, dp(v["d"]), dp(v["u"]), dp(v["l"]), hasA)),
                        {"sf": sf}, (), {"d": A["diag"], "u": np.zeros(1), "l": np.zeros(1)})
    for mode in (0, 1, 2):
        r[f"rs{mode}"] = D.call(lambda v: capi.check(L.b200ldu_ldu_row_sum(a, mode, dp(v["u"]), dp(v["l"]), dp(v["io"]))),
                                {"u": np.zeros(1), "l": np.zeros(1)}, (), {"io": A["diag"]})["io"]
    D.close()
    return r


def test_ldu_algebra_without_faces(gpu):
    """lduMatrix += -= *= and the row sums on a 1-cell addressing: only the diagonal changes (the face arrays, one unused double
    each, are written by nothing)"""
    box = hc.build("cell1")
    A, B, sf = dict(diag=np.array([1.5])), dict(diag=np.array([0.25])), np.array([3.0])
    r = both(gpu, lambda capi, ctx, torch: _ldu_no_faces(capi, ctx, torch, box, A, B, sf))
    assert r["aa0"]["d"][0] == 1.75 and r["aa1"]["d"][0] == 1.25
    assert r["scale"]["d"][0] == 4.5
    assert r["rs0"][0] == 1.5 and r["rs1"][0] == 1.5 and r["rs2"][0] == 1.5
    for k in ("aa0", "aa1", "scale"):
        assert (r[k]["u"] == 0).all() and (r[k]["l"] == 0).all(), k


# ---- d. field operators --------------------------------------------------------------------------------------------------
FIELD_N = [0, 1, 2, 3, 255, 256, 257]
NC_MIX = [(1, 1), (1, 3), (3, 1), (3, 3)]


def field_inputs(n, seed=9):
    rng = np.random.default_rng(seed + n)
    a3, b3 = rng.uniform(-2, 2, 3 * n), rng.uniform(0.5, 2, 3 * n) * rng.choice([-1.0, 1.0], 3 * n)
    a3[::5] = 0.0
    a3[1::7] = -0.0
    return dict(a1=a3[:n].copy(), a3=a3, b1=b3[:n].copy(), b3=b3, T=rng.uniform(-1, 1, 9 * n), cells=rng.integers(0, max(n, 1), n))


def binary_reference(op, A, B, nca, ncb):
    a, b = A.reshape(-1, nca), B.reshape(-1, ncb)
    return np.ravel([np.add, np.subtract, np.multiply, np.divide, fo.min_, fo.max_][op](a, b))


def unary_reference(op, a, s):
    with np.errstate(divide="ignore"):
        return [-a, np.abs(a), s * a, s / a, a + s, s - a, fo.min_(a, s), fo.max_(a, s), a - s, a / s, a.copy(),
                np.where(a >= 0, 1.0, 0.0)][op]


def _fields(capi, ctx, torch, n, I):
    L, dp, h = capi.lib(), capi._dp, ctx.h
    c = lambda fn, ins, outs: call(torch, ctx.device, fn, ins, outs)
    r = {}
    for op in range(6):
        for nca, ncb in NC_MIX:
            nc = max(nca, ncb)
            r[f"b{op}{nca}{ncb}"] = c(lambda v: capi.check(L.b200ldu_field_binary(h, op, n, nca, dp(v["a"]), ncb, dp(v["b"]), dp(v["o"]))),
                                      {"a": I[f"a{nca}"], "b": I[f"b{ncb}"]}, {"o": n * nc})["o"]
    for op in range(12):
        r[f"u{op}"] = c(lambda v: capi.check(L.b200ldu_field_unary(h, op, 3 * n, -1.25, dp(v["a"]), dp(v["o"]))), {"a": I["a3"]},
                        {"o": 3 * n})["o"]
    r["dot3"] = c(lambda v: capi.check(L.b200ldu_field_dot3(h, n, dp(v["a"]), dp(v["b"]), dp(v["o"]))), {"a": I["a3"], "b": I["b3"]},
                  {"o": n})["o"]
    r["symm"] = c(lambda v: capi.check(L.b200ldu_field_symm_magsqr(h, n, dp(v["T"]), dp(v["o"]))), {"T": I["T"]}, {"o": n})["o"]
    cells = torch.from_numpy(np.ascontiguousarray(np.concatenate([I["cells"], [0]]), np.int32)).to(ctx.device)
    for nc in (1, 3):
        r[f"g{nc}"] = c(lambda v: capi.check(L.b200ldu_field_gather(h, n, nc, dp(cells), dp(v["f"]), dp(v["o"]))), {"f": I[f"a{nc}"]},
                        {"o": n * nc})["o"]
    return r


@pytest.mark.parametrize("n", FIELD_N)
def test_field_operators(gpu, n):
    from oracle import kepsilon_oracle as ko
    I = field_inputs(n)
    r = both(gpu, lambda capi, ctx, torch: _fields(capi, ctx, torch, n, I))
    for op in range(6):
        for nca, ncb in NC_MIX:
            assert np.array_equal(bits(r[f"b{op}{nca}{ncb}"]), bits(binary_reference(op, I[f"a{nca}"], I[f"b{ncb}"], nca, ncb))), (op, nca, ncb)
    for op in range(12):
        assert np.array_equal(bits(r[f"u{op}"]), bits(unary_reference(op, I["a3"], -1.25))), op
    A, B = I["a3"].reshape(-1, 3), I["b3"].reshape(-1, 3)
    assert np.array_equal(r["dot3"], (A[:, 0] * B[:, 0] + A[:, 1] * B[:, 1]) + A[:, 2] * B[:, 2])
    assert np.array_equal(r["symm"], np.ravel(ko.symm_magsqr(I["T"].reshape(-1, 9))))
    for nc in (1, 3):
        assert np.array_equal(r[f"g{nc}"], I[f"a{nc}"].reshape(-1, nc)[I["cells"]].ravel()), nc


# ---- e. reuse after growth -----------------------------------------------------------------------------------------------
def _small(capi, ctx, torch, box, sym, asym, x, b):
    D = Dev(capi, ctx, torch, box, sym)
    h, L, dp = D.mat.h, D.L, D.dp
    amul = lambda: D.call(lambda v: capi.check(L.b200ldu_amul(h, dp(v["x"]), dp(v["y"]))), {"x": x}, {"y": box.nCells})["y"]
    tmul = lambda: D.call(lambda v: capi.check(L.b200ldu_tmul(h, dp(v["x"]), dp(v["y"]))), {"x": x}, {"y": box.nCells})["y"]
    r = {"sym": (amul(), _solve(D, "PCG", "DIC", x, b, tolerance=1e-9)[1:])}
    D.set(asym)          # a second coefficient stream for Tmul (MAT_VALT grows)
    r["asym"] = (amul(), tmul(), _solve(D, "PBiCGStab", "DILU", x, b, tolerance=1e-9)[1:])
    D.set(sym)
    r["sym2"] = amul()
    for cap in (4, 32, 512):                                      # the device residual history grows (MAT_HIST)
        r[f"hist{cap}"] = _solve(D, "PCG", "DIC", x, b, histCap=cap, tolerance=0.0, maxIter=60)[1:]
    D.close()
    return r


def test_reuse_after_growth(gpu, orc, meshmod):
    capi, ctxs, torch = gpu
    big = meshmod.hex_mesh(40, 40, 40)
    c = meshmod.pressure_laplacian(big)
    A = capi.mesh_to_device(ctxs[True], big)
    M = capi.LduMatrix(A)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(ctxs[True].device)
    M.set(t(c["diag"]), t(c["upper"]))
    psi = torch.zeros(big.nCells, dtype=torch.float64, device=ctxs[True].device)
    perf, _ = M.solve("PCG", "DIC", psi, t(meshmod.cell_field_global(big, 3)), tolerance=1e-8, maxIter=50)
    assert perf.nIterations >= 50
    M.close()
    A.close()
    box = hc.build("chain129")
    sym = hc.coefficients(box, True, 2)
    asym = hc.coefficients(box, False, 2)
    rng = np.random.default_rng(3)
    x, b = rng.uniform(-1, 1, box.nCells), rng.uniform(-1, 1, box.nCells)
    reused = _small(capi, ctxs[True], torch, box, sym, asym, x, b)
    with environ(**{POISON: "1"}):
        fresh_ctx = capi.Context(0)
    try:
        fresh = _small(capi, fresh_ctx, torch, box, sym, asym, x, b)
    finally:
        fresh_ctx.close()
    same(reused, fresh)
    _, om = hc.oracle_matrix(orc, box, sym)
    _, oma = hc.oracle_matrix(orc, box, asym)
    assert np.array_equal(reused["sym"][0], om.amul(x)) and np.array_equal(reused["sym2"], om.amul(x))
    assert np.array_equal(reused["asym"][0], oma.amul(x)) and np.array_equal(reused["asym"][1], oma.tmul(x))
    hs = [reused[f"hist{cap}"][2] for cap in (4, 32, 512)]
    assert len(hs[0]) == 4 and len(hs[1]) == 32
    assert np.array_equal(hs[0], hs[2][:4]) and np.array_equal(hs[1], hs[2][:32])


# ---- f. multi-GPU --------------------------------------------------------------------------------------------------------
def test_multi_gpu_poisoned():
    """tests/multi_gpu_worker.py (halo exchange, all-reduce and GAMG over processor patches) on two GPUs with every new block of the
    library poisoned"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29652", os.path.join(ROOT, "tests", "multi_gpu_worker.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, MASTER_ADDR="127.0.0.1", **{POISON: "1"}), capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-4000:]
    assert p.stdout.count("MULTI-GPU-OK") == 9
