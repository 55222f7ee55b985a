"""The banded engine's two streams on the device.  A symmetric matrix runs on the face stream (FS: every face stored
once, the transposed products added from a shared-memory buffer) when its layout has one; everything else runs on
the entry stream (ES: every row's entries stored in full).  B200LDU_FACE_STREAM=0 / =1 pick the stream and
B200LDU_BAND_ROWS the band size when an addressing (or a GAMG hierarchy and its coarse levels) is built, so one mesh is
built twice and the two streams are compared with each other BIT FOR BIT (int64 views: -0.0 != +0.0), and each with
the oracle wherever DESIGN.md section 2 states bit equality.

The cases reach what small one-wave meshes do not: bands of several slices (several warps in both passes, slice
loops past the eighth slice at 1024 and 2048 rows, in-band products stored into another slice's buffer), more than
40 KB of dynamic shared memory, bands narrowed on a graph without locality, and coupled (cyclic) patches whose matrix
shares one array for interfaceBouCoeffs and interfaceIntCoeffs -- the only way a matrix with interfaces keeps the
face stream."""
import contextlib
import importlib
import math
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BAND_ENV, FS_ENV = "B200LDU_BAND_ROWS", "B200LDU_FACE_STREAM"


@contextlib.contextmanager
def environ(**kv):
    """Sets (value) or unsets (None) environment variables for the duration of the block, then restores them."""
    old = {k: os.environ.get(k) for k in kv}
    try:
        for k, v in kv.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def engine_env(band=None, fs=None):
    """Band size and stream choice, both read by the layout builder when an addressing is created."""
    return environ(**{BAND_ENV: band, FS_ENV: fs})


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


class Mismatches:
    """Collects every failed comparison of a test, so that one failure report shows all of them."""

    def __init__(self):
        self.msgs = []

    def bits(self, got, ref, what):
        got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
        if got.shape != ref.shape:
            self.msgs.append(f"{what}: shape {got.shape} != {ref.shape}")
            return
        bad = np.nonzero(bits(got) != bits(ref))[0]
        if len(bad):
            zs = np.count_nonzero((got[bad] == 0) & (ref[bad] == 0))
            self.msgs.append(f"{what}: {len(bad)} of {len(got)} differ ({zs} only in the sign of a zero), first rows "
                             f"{bad[:4].tolist()}: {got[bad[:4]].tolist()} vs {ref[bad[:4]].tolist()}")

    def bits_es(self, es, ref, what):
        """`es` from the entry stream: bit for bit, except the stated exception (DESIGN.md section 4) -- a padding
        slot adds prod(0, a_own), so a row whose terms sum to -0 may come out +0 (never anything else)"""
        es, ref = np.asarray(es, np.float64), np.asarray(ref, np.float64)
        if es.shape == ref.shape:
            es = np.where((bits(es) == 0) & (bits(ref) == bits(np.array(-0.0))), ref, es)
        self.bits(es, ref, what)

    def close(self, got, ref, what, rtol):
        try:
            np.testing.assert_allclose(got, ref, rtol=rtol, atol=rtol * float(np.max(np.abs(ref), initial=0.0)))
        except AssertionError as e:
            self.msgs.append(f"{what}: {str(e).strip().splitlines()[-1]}")

    def true(self, ok, what):
        if not ok:
            self.msgs.append(what)

    def check(self):
        assert not self.msgs, f"{len(self.msgs)} mismatch(es):\n" + "\n".join(self.msgs)


# ---- problems: addressing, symmetric coefficients, oracle ---------------------------------------------------------
class Problem:
    def __init__(self, orc, nCells, lower, upper, diag, up, centres=None, patches=None, bou=None, mesh=None,
                 meshmod=None, parity=None, seed=0):
        self.orc, self.meshmod = orc, meshmod
        self.nCells, self.lower, self.upper = nCells, np.asarray(lower, np.int32), np.asarray(upper, np.int32)
        self.nFaces = len(self.lower)
        self.diag, self.up, self.bou = diag, up, bou
        self.centres, self.mesh, self.seed = centres, mesh, seed
        self.ps, self.fc, self.nr = patches if patches is not None else (None, None, None)
        self.periodic = patches is not None
        # sign pattern of the signed-zero input: a row whose own value is +0 and whose neighbours are all -0 sums to
        # -0 with a negative diagonal and positive off-diagonals (the OpenFOAM sign of a Laplacian)
        self.parity = parity if parity is not None else np.random.default_rng(seed + 99).integers(0, 2, nCells)
        if self.periodic:
            self.oa = orc.Addr(nCells, self.lower, self.upper, self.ps, self.fc, neighbRank=self.nr)
        else:
            self.oa = orc.Addr(nCells, self.lower, self.upper)
        self.om = self.oracle_matrix(diag, up)

    def oracle_matrix(self, diag, up, lower=None, bou=None, intc=None):
        if self.periodic:
            bou = self.bou if bou is None else bou
            return self.orc.Matrix(self.oa, diag, up, lower, bou, bou if intc is None else intc)
        return self.orc.Matrix(self.oa, diag, up, lower)

    def field(self, seed):
        if self.mesh is not None:
            return self.meshmod.cell_field_global(self.mesh, seed)
        return np.random.default_rng(seed).uniform(-1.0, 1.0, self.nCells)

    def signed_zeros(self, seed):
        """blocks of exact +0.0 / -0.0 (signs from the parity pattern, or all +0, or all -0) between blocks of
        ordinary values"""
        x = self.field(seed)
        # slabs of several mesh layers, so that whole neighbourhoods carry the pattern
        blk = (np.arange(self.nCells) // max(41, self.nCells // 12) + seed) % 4
        par = np.where(self.parity == 1, -0.0, 0.0)
        x = np.where(blk == 0, par, x)
        x = np.where(blk == 1, 0.0, x)
        x = np.where(blk == 2, -0.0, x)
        x[: min(self.nCells, 3)] = par[: min(self.nCells, 3)]  # the tiny meshes have no block 0 otherwise
        return x

    def wide(self, seed):
        """magnitudes spread over 1e-150 .. 1e150, random signs"""
        rng = np.random.default_rng(seed)
        return rng.choice([-1.0, 1.0], self.nCells) * 10.0 ** rng.uniform(-150, 150, self.nCells)


def _hex_parity(m):
    c = np.arange(m.nCells)
    return ((c % m.nx) + (c // m.nx) % m.ny + c // (m.nx * m.ny)) % 2


def hex_problem(meshmod, orc, dims, centres=True):
    m = meshmod.hex_mesh(*dims)
    c = meshmod.pressure_laplacian(m)
    diag = c["diag"]
    if m.nCells == 1:
        diag = np.array([-1.0])  # a lone pinned cell has no coefficients: its diagonal would be 0
    return Problem(orc, m.nCells, m.lower, m.upper, diag, c["upper"], m.cell_centres() if centres else None, mesh=m,
                   meshmod=meshmod, parity=_hex_parity(m))


def periodic_problem(meshmod, orc, dims):
    """hex box periodic in x: the x-min and x-max wall faces become a cyclic patch pair (neighbRank -(partner+1)),
    pressure-Laplacian coefficients on the new faces; one array serves as bou and int coefficients"""
    nx, ny, nz = dims
    m = meshmod.hex_mesh(nx, ny, nz)
    c = meshmod.pressure_laplacian(m, pin=False)
    jk = np.arange(ny * nz)
    lo = (jk * nx).astype(np.int32)
    hi = (jk * nx + nx - 1).astype(np.int32)
    coeff = np.random.default_rng(5).uniform(0.5, 1.5, ny * nz) * m.h
    diag = c["diag"].copy()
    np.subtract.at(diag, lo, coeff)
    np.subtract.at(diag, hi, coeff)
    diag[0] *= 2  # pin (setReference)
    bou = np.concatenate([-coeff, -coeff])
    patches = (np.array([0, ny * nz, 2 * ny * nz], np.int32), np.concatenate([lo, hi]).astype(np.int32),
               np.array([-2, -1], np.int32))
    return Problem(orc, m.nCells, m.lower, m.upper, diag, c["upper"], m.cell_centres(), patches=patches, bou=bou,
                   mesh=m, meshmod=meshmod, parity=_hex_parity(m))


def random_problem(orc, k):
    """random graph without locality (no centres): symmetric coefficients of both signs, negative and diagonally
    dominant diagonal"""
    from test_layout_cpu import _RandomGraph
    g = _RandomGraph(30000, k, 1)
    rng = np.random.default_rng(17)
    up = rng.uniform(-1.0, 1.0, g.nFaces)
    s = np.zeros(g.nCells)
    np.add.at(s, g.lower, np.abs(up))
    np.add.at(s, g.upper, np.abs(up))
    diag = -(s + 0.1) * rng.uniform(1.0, 1.5, g.nCells)
    return Problem(orc, g.nCells, g.lower, g.upper, diag, up, seed=3)


# case name -> (builder, band sizes); None = the library's own choice
CASES = {
    "hex40x24x20": (lambda mm, o: hex_problem(mm, o, (40, 24, 20)), (64, 128, 256, 512, 1024, 2048)),
    "hex37x23x11_nocentres": (lambda mm, o: hex_problem(mm, o, (37, 23, 11), centres=False), (512,)),
    "hex1": (lambda mm, o: hex_problem(mm, o, (1, 1, 1)), (None,)),
    "hex3x1x1": (lambda mm, o: hex_problem(mm, o, (3, 1, 1)), (None,)),
    # 16384 rows asked, narrowed to 1024 (the halo of a band takes ~8000 columns): the face stream then needs 182 KB of
    # shared memory.  The 6-faces-per-cell graph of the CPU layout tests narrows to 1024 rows too, but its face stream
    # would need 243 KB and cannot fit (test_face_stream_does_not_fit)
    "random30000": (lambda mm, o: random_problem(o, 4), (16384,)),
    "periodic24x20x16": (lambda mm, o: periodic_problem(mm, o, (24, 20, 16)), (64, 256, 512)),
    "hex128": (lambda mm, o: hex_problem(mm, o, (128, 128, 128)), (None,)),
}
PARAMS = [pytest.param(name, band, id=f"{name}-{band or 'default'}") for name, (_, bands) in CASES.items()
          for band in bands]
SOLVER_PARAMS = [p for p in PARAMS if p.values[0] not in ("hex1",)]
LARGE = "hex128"


# ---- device side ---------------------------------------------------------------------------------------------------
class Side:
    """One addressing + matrix of a problem on one stream."""

    def __init__(self, gpu, pb, band, fs):
        capi, ctx, torch = gpu
        self.capi, self.ctx, self.torch, self.pb, self.band, self.fs = capi, ctx, torch, pb, band, fs
        with engine_env(band, fs):
            self.addr = capi.LduAddressing(ctx, pb.nCells, pb.lower, pb.upper, pb.ps, pb.fc, pb.nr, pb.centres)
        self.info = self.addr.info()
        self.mat = capi.LduMatrix(self.addr)
        self.set(pb.diag, pb.up)

    def t(self, a):
        if a is None or len(a) == 0:
            return None
        return self.torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(self.ctx.device)

    def set(self, diag, up, lower=None, bou=None, intc=None):
        """symmetric unless `lower`; interfaces: ONE tensor for both coefficient arrays unless `intc` is given"""
        b = None
        if self.pb.periodic:
            b = self.t(self.pb.bou if bou is None else bou)
        i = b if intc is None else self.t(intc)
        self.keep = (self.t(diag), self.t(up), self.t(lower), b, i)
        self.mat.set(*self.keep)

    def zeros(self):
        return self.torch.zeros(self.pb.nCells, dtype=self.torch.float64, device=self.ctx.device)

    def gamg(self, weights, nCoarsest=10):
        with engine_env(self.band, self.fs):  # the coarse levels' layouts follow the finest level's stream
            return self.capi.GamgAgglomeration(self.addr, weights, nCoarsest, 1)

    def close(self):
        self.mat.close()
        self.addr.close()


def smem_kb_min(info):
    """lower bound of a face-stream sweep's dynamic shared memory (the halo part of the tile is not in info())"""
    return 8 * (info["bandRows"] + info["fsBufDoubles"]) / 1024


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available()
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


@pytest.fixture(scope="module")
def cases(gpu, meshmod, orc):
    """(problem, ES side, FS side) per (case, band), built once for the module"""
    problems, built = {}, {}

    def pair(name, band):
        if (name, band) not in built:
            if name not in problems:
                problems[name] = CASES[name][0](meshmod, orc)
            pb = problems[name]
            es, fs = Side(gpu, pb, band, 0), Side(gpu, pb, band, 1)
            # no case may silently compare the entry stream with itself
            assert not es.info["faceStream"], (name, band, es.info)
            assert fs.info["faceStream"], (name, band, fs.info)
            assert es.info["bandRows"] == fs.info["bandRows"] and es.info["nBands"] == fs.info["nBands"]
            if pb.centres is None and pb.mesh is None:
                assert fs.info["bandRows"] < band  # the random graph's bands were narrowed
            i = fs.info
            print(f"\n[engine-streams] {name} band={band}: bandRows={i['bandRows']} nBands={i['nBands']} "
                  f"fsBufDoubles={i['fsBufDoubles']} smem>={smem_kb_min(i):.1f}KB "
                  f"(>40KB: {'yes' if smem_kb_min(i) > 40 else 'check'})")
            built[(name, band)] = (pb, es, fs)
        return built[(name, band)]

    yield pair
    for pb, es, fs in built.values():
        es.close()
        fs.close()


# ---- operators -----------------------------------------------------------------------------------------------------
def _ops(side, x, b):
    """every row-gather operation on (x, b), host arrays by name"""
    xd, bd = side.t(x), side.t(b)
    m = side.mat
    out = {"Amul": m.Amul(xd), "Tmul": m.Tmul(xd), "residual": m.residual(xd, bd), "H": m.H(xd)}
    if side.pb.nFaces:
        out["faceH"] = m.faceH(xd)
    for pre in ("none", "diagonal", "DIC"):
        for T in (False, True):
            out[f"precondition-{pre}-T{int(T)}"] = m.precondition(pre, xd, T)
    for ns in (1, 2, 3):
        out[f"GaussSeidel-{ns}"] = m.smooth("GaussSeidel", xd, bd, ns)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _ops_oracle(om, x, b, large):
    ref = {"Amul": om.amul(x), "residual": om.residual(x, b)}
    ref["precondition-DIC-T0"] = om.precondition("DIC", x, False)
    if large:  # 2 M cells: the oracle side is trimmed to Amul, residual and AINV
        return ref
    ref.update({"Tmul": om.tmul(x), "H": om.H(x)})
    if om.addr.nFaces:
        ref["faceH"] = om.faceH(x)
    for pre in ("none", "diagonal", "DIC"):
        for T in (False, True):
            ref[f"precondition-{pre}-T{int(T)}"] = om.precondition(pre, x, T)
    for ns in (1, 2, 3):
        ref[f"GaussSeidel-{ns}"] = om.jacobi(x, b, ns)
    return ref


def _inputs(pb):
    return [("field", pb.field(3), pb.field(4)), ("signed-zeros", pb.signed_zeros(5), pb.signed_zeros(6)),
            ("wide", pb.wide(7), pb.wide(8))]


@pytest.mark.parametrize("name,band", PARAMS)
def test_operators(cases, name, band):
    """Amul, Tmul, sumA, residual, H, H1, faceH, precondition none / diagonal / DIC (plain and transposed) and
    GaussSeidel with 1-3 sweeps: the face stream bit for bit the entry stream, both bit for bit the oracle except the
    stated exceptions (AINV's association, Jacobi with coupled interfaces: 1e-13)."""
    pb, es, fs = cases(name, band)
    large = name == LARGE
    M = Mismatches()
    like = es.zeros()
    for nm, side in (("ES", es), ("FS", fs)):
        s, h1 = side.mat.sumA(like).cpu().numpy(), side.mat.H1(like).cpu().numpy()
        if side is es:
            sES, h1ES = s, h1
        else:
            M.bits(s, sES, "sumA FS vs ES")
            M.bits(h1, h1ES, "H1 FS vs ES")
        if not large:
            M.bits(s, pb.om.sumA(), f"sumA {nm} vs oracle")
            M.bits(h1, pb.om.H1(), f"H1 {nm} vs oracle")
    for inp, x, b in _inputs(pb):
        got = {"ES": _ops(es, x, b), "FS": _ops(fs, x, b)}
        ref = _ops_oracle(pb.om, x, b, large)
        for op, v in got["FS"].items():
            M.bits_es(got["ES"][op], v, f"{op} [{inp}] ES vs FS")
        for nm in ("ES", "FS"):
            for op, r in ref.items():
                v, what = got[nm][op], f"{op} [{inp}] {nm} vs oracle"
                if op.startswith("precondition-DIC") or (op.startswith("GaussSeidel") and pb.periodic):
                    M.close(v, r, what, 1e-13)
                elif nm == "ES":
                    M.bits_es(v, r, what)
                else:
                    M.bits(v, r, what)
    M.check()


# ---- solvers -------------------------------------------------------------------------------------------------------
def _solve(side, solver, pre, b, psi0=None, gamg=None, fused=None, **ctl):
    psi = side.zeros() if psi0 is None else side.t(psi0)
    with environ(B200LDU_PCG_FUSED=fused):
        perf, hist = side.mat.solve(solver, pre, psi, side.t(b), gamg=gamg, histCap=2048, **ctl)
    return perf, hist, psi.cpu().numpy()


def _same_solve(M, a, b, what):
    (pa, ha, xa), (pb_, hb, xb) = a, b
    M.true(pa.nIterations == pb_.nIterations and pa.converged == pb_.converged,
           f"{what}: nIterations/converged FS {pb_.nIterations}/{pb_.converged} vs ES {pa.nIterations}/{pa.converged}")
    M.bits(hb, ha, f"{what}: history FS vs ES")
    M.bits(xb, xa, f"{what}: psi FS vs ES")
    for k in ("initialResidual", "finalResidual", "normFactor"):
        M.bits([getattr(pb_, k)], [getattr(pa, k)], f"{what}: {k} FS vs ES")


def _vs_oracle(M, got, ref, what, rtol=1e-9, first=30):
    perf, hist, _ = got
    _, pr, href = ref
    # the documented contract: identical counts, +-1 beyond 100 iterations (the global sums' order differs)
    M.true(abs(perf.nIterations - pr.nIterations) <= (0 if pr.nIterations < 100 else 1),
           f"{what}: nIterations {perf.nIterations} vs oracle {pr.nIterations}")
    k = min(first, len(hist), len(href))
    M.close(hist[:k], href[:k], f"{what}: history vs oracle", rtol)


@pytest.mark.parametrize("name,band", SOLVER_PARAMS)
def test_solvers(cases, meshmod, orc, name, band):
    """PCG (DIC, diagonal, none; fused and the op-list path; 25 fixed iterations and a converging run), smoothSolver
    and GAMG: psi, history and counts byte-identical between the streams, history to 1e-9 (GAMG 1e-8) and the same
    counts as the oracle."""
    pb, es, fs = cases(name, band)
    large = name == LARGE
    M = Mismatches()
    b = pb.om.amul(pb.field(42))
    for pre in ("DIC", "diagonal", "none"):
        for ctl in (dict(tolerance=0.0, maxIter=25), dict(tolerance=1e-8, maxIter=1000)):
            # 2 M cells: the oracle runs 30 DIC iterations only
            ref = None
            if not large:
                ref = pb.om.solve("PCG", pre, np.zeros(pb.nCells), b, **ctl)
            elif pre == "DIC" and ctl["tolerance"] == 0.0:
                ref = pb.om.solve("PCG", pre, np.zeros(pb.nCells), b, tolerance=0.0, maxIter=30)
                ctl = dict(tolerance=0.0, maxIter=30)
            for fused in ("1", "0"):
                what = f"PCG {pre} {ctl} fused={fused}"
                r_es = _solve(es, "PCG", pre, b, fused=fused, **ctl)
                r_fs = _solve(fs, "PCG", pre, b, fused=fused, **ctl)
                _same_solve(M, r_es, r_fs, what)
                if ref is not None:
                    _vs_oracle(M, r_fs, ref, what)
    if pb.periodic:
        # Jacobi with coupled interfaces: the stated 1e-13 per sweep, measured 3e-8 on the cycle residuals of a
        # 120-cell box (test_gpu_parity.test_cyclic_interfaces)
        rtol_j, first_j = 1e-6, 10
    else:
        rtol_j, first_j = 1e-9, 30
    ctl = dict(tolerance=0.0, maxIter=40, nSweeps=2)
    r_es, r_fs = (_solve(s, "smoothSolver", "GaussSeidel", b, **ctl) for s in (es, fs))
    _same_solve(M, r_es, r_fs, "smoothSolver 2 sweeps")
    if not large:
        _vs_oracle(M, r_fs, pb.om.solve("smoothSolver", "GaussSeidel", np.zeros(pb.nCells), b, **ctl),
                   "smoothSolver 2 sweeps", rtol_j, first_j)
    if name == "hex40x24x20" and band in (64, 512) or pb.periodic:
        w = meshmod.face_area_pair_weights(pb.mesh)
        og = orc.Gamg(pb.oa, w, 10, 1)
        ctl = dict(tolerance=1e-9, maxIter=100)
        ref = og.solve(pb.om, "GaussSeidel", np.zeros(pb.nCells), b, **ctl)
        res = []
        for side in (es, fs):
            gg = side.gamg(w)
            M.true(gg.nLevels == og.nLevels, f"GAMG levels {gg.nLevels} vs oracle {og.nLevels}")
            res.append(_solve(side, "GAMG", "GaussSeidel", b, gamg=gg, **ctl))
            gg.close()
        _same_solve(M, res[0], res[1], "GAMG")
        _vs_oracle(M, res[1], ref, "GAMG", 1e-6 if pb.periodic else 1e-8, first=len(ref[2]))
        M.true(res[1][0].converged == 1, "GAMG did not converge")
    M.check()


# ---- reductions against an exactly rounded sum ---------------------------------------------------------------------
# Measured on one H100 80GB HBM3 (400 W power limit) over every case and band size below: 0 (both quantities equal the exactly rounded sum).
# The terms are all positive, so any grouping is within (depth of the summation tree) * 2^-53 of it: ~30 levels for
# 2 M cells, 3.3e-15; the tolerance allows three times that.
REDUCTION_RTOL = 1e-14


@pytest.mark.parametrize("name,band", SOLVER_PARAMS)
def test_reductions_against_fsum(cases, name, band):
    """normFactor and initialResidual of a maxIter=0 PCG solve from a non-zero psi, against math.fsum of the same
    |.| terms (lduMatrixSolver.C:183-236 with the oracle's A psi and sumA): the band size regroups the per-block
    partial sums, both streams share that code."""
    pb, es, fs = cases(name, band)
    psi0 = pb.field(11)
    b = pb.field(12)
    Apsi, sA = pb.om.amul(psi0), pb.om.sumA()
    t = (math.fsum(psi0) / pb.nCells) * sA
    nf = math.fsum(np.concatenate([np.abs(Apsi - t), np.abs(b - t)])) + 1e-20
    ir = math.fsum(np.abs(b - Apsi)) / nf
    M = Mismatches()
    got = [_solve(s, "PCG", "DIC", b, psi0=psi0, tolerance=0.0, maxIter=0) for s in (es, fs)]
    _same_solve(M, got[0], got[1], "PCG maxIter=0")
    perf = got[1][0]
    e_nf, e_ir = abs(perf.normFactor - nf) / nf, abs(perf.initialResidual - ir) / ir
    print(f"\n[engine-streams] reductions {name} band={band}: normFactor rel {e_nf:.2e}, initialResidual rel {e_ir:.2e}")
    M.true(e_nf <= REDUCTION_RTOL, f"normFactor {perf.normFactor!r} vs fsum {nf!r}: rel {e_nf:.3e}")
    M.true(e_ir <= REDUCTION_RTOL, f"initialResidual {perf.initialResidual!r} vs fsum {ir!r}: rel {e_ir:.3e}")
    M.check()


def test_benchmark_regime(gpu, meshmod, orc):
    """128^3 without overrides (the benchmark's mesh): 512-row bands and the face stream"""
    m = meshmod.hex_mesh(128)
    capi, ctx, _ = gpu
    with engine_env(None, None):
        addr = capi.mesh_to_device(ctx, m)
    info = addr.info()
    addr.close()
    assert info["bandRows"] == 512 and info["faceStream"], info


def test_face_stream_does_not_fit(gpu):
    """The expected exception: B200LDU_FACE_STREAM=1 keeps the entry stream where the product buffer does not fit next
    to the tile (a random graph with ~12 faces per cell: 1024-row bands after narrowing, 243 KB)"""
    from test_layout_cpu import _RandomGraph
    capi, ctx, _ = gpu
    g = _RandomGraph(30000, 6, 1)
    with engine_env(16384, 1):
        addr = capi.LduAddressing(ctx, g.nCells, g.lower, g.upper)
    info = addr.info()
    addr.close()
    assert info["bandRows"] < 16384 and not info["faceStream"], info


# ---- matrix re-set on one addressing -------------------------------------------------------------------------------
def _reset_step(M, side, witness, om, inputs, b, expect_fs, what):
    """`side` is the face-stream addressing after a set, `witness` an entry-stream addressing of the same mesh and band
    set with the same coefficients.  Running the face stream, `side` gives the oracle's bits and differs from the
    witness in the sign of some zero row sums of the signed-zero input (the entry stream's padding); running the
    entry stream, it gives the witness's bits."""
    differs = False
    for x in inputs:
        xd, bd, xw, bw = side.t(x), side.t(b), witness.t(x), witness.t(b)
        for op, got, wit, ref in (("Amul", side.mat.Amul(xd), witness.mat.Amul(xw), om.amul(x)),
                                  ("Tmul", side.mat.Tmul(xd), witness.mat.Tmul(xw), om.tmul(x)),
                                  ("residual", side.mat.residual(xd, bd), witness.mat.residual(xw, bw),
                                   om.residual(x, b))):
            got, wit = got.cpu().numpy(), wit.cpu().numpy()
            if expect_fs:
                M.bits(got, ref, f"{what}: {op} vs oracle")
            else:
                M.bits(got, wit, f"{what}: {op} vs the entry stream")
                M.bits_es(got, ref, f"{what}: {op} vs oracle")
            differs |= not np.array_equal(bits(got), bits(wit))
    M.true(differs == expect_fs, f"{what}: the results {'differ from' if differs else 'equal'} the entry stream's")


def test_matrix_reset_hex(gpu, meshmod, orc):
    """One face-stream addressing, set in turn with P, U (asymmetric: entry stream), P, 3 P: the coefficient storage
    switches each time, the stream follows, every result is the oracle's."""
    pb = hex_problem(meshmod, orc, (16, 12, 10))
    side, witness = Side(gpu, pb, 128, 1), Side(gpu, pb, 128, 0)
    assert side.info["faceStream"] and side.info["bandRows"] == 128, side.info
    mom = meshmod.momentum_matrix(pb.mesh)
    M = Mismatches()
    inputs, b = (pb.signed_zeros(1), pb.field(3)), pb.field(2)
    steps = [("P", (pb.diag, pb.up, None)), ("U", (mom["diag"], mom["upper"], mom["lower"])),
             ("P again", (pb.diag, pb.up, None)), ("3 P", (3 * pb.diag, 3 * pb.up, None))]
    for what, (d, u, lo) in steps:
        side.set(d, u, lo)
        witness.set(d, u, lo)
        _reset_step(M, side, witness, pb.oracle_matrix(d, u, lo), inputs, b, lo is None, what)
        if lo is not None:  # the asymmetric matrix runs with its own transpose
            x = side.t(inputs[1])
            M.true(not torch_equal(side.mat.Tmul(x), side.mat.Amul(x)), f"{what}: Tmul == Amul")
    side.close()
    witness.close()
    M.check()


def torch_equal(a, b):
    return np.array_equal(bits(a.cpu().numpy()), bits(b.cpu().numpy()))


def test_matrix_reset_periodic(gpu, meshmod, orc):
    """One face-stream addressing with cyclic patches, set with one interface array (face stream), two distinct
    arrays with different values (entry stream with its own transpose: Tmul != Amul), then one array again.  Callers
    that pass equal but distinct arrays get the entry stream: the choice compares the pointers."""
    pb = periodic_problem(meshmod, orc, (24, 20, 16))
    side, witness = Side(gpu, pb, 256, 1), Side(gpu, pb, 256, 0)
    assert side.info["faceStream"], side.info
    M = Mismatches()
    inputs, b = (pb.signed_zeros(5), pb.field(3)), pb.field(4)
    n = len(pb.bou) // 2
    skew = np.concatenate([0.5 * pb.bou[:n], 1.5 * pb.bou[n:]])
    skewT = np.concatenate([1.5 * pb.bou[:n], 0.5 * pb.bou[n:]])
    for what, bou, intc in (("shared", pb.bou, None), ("distinct", skew, skewT), ("shared again", pb.bou, None)):
        side.set(pb.diag, pb.up, None, bou, intc)
        witness.set(pb.diag, pb.up, None, bou, intc)
        om = pb.oracle_matrix(pb.diag, pb.up, None, bou, bou if intc is None else intc)
        _reset_step(M, side, witness, om, inputs, b, intc is None, what)
        x = side.t(inputs[1])
        same = torch_equal(side.mat.Tmul(x), side.mat.Amul(x))
        M.true(same == (intc is None), f"{what}: Tmul == Amul is {same}")
    side.close()
    witness.close()
    M.check()
