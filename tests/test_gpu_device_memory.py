"""Device memory of the library's handles, read through b200ldu_ctx_device_mem: every handle gives back what it
allocated, a create that fails leaves nothing behind, the solver and fvMatrix entry points allocate nothing once
warmed up, and a matrix that switches between the symmetric and the asymmetric coefficient stream keeps only the one
it uses."""
import ctypes as C
import importlib

import numpy as np
import pytest

from test_mules_cpu import case as mules_case
from test_oracle_fvm import momentum_case, poisson_case

pytestmark = pytest.mark.gpu

DIMS = (12, 10, 8)


@pytest.fixture(scope="module")
def gpu():
    import torch
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


def device_mem(capi, ctx):
    live, n = C.c_longlong(), C.c_longlong()
    capi.check(capi.lib().b200ldu_ctx_device_mem(ctx.h, C.byref(live), C.byref(n)))
    return live.value, n.value


def tensor(ctx, torch, a):
    return torch.from_numpy(np.array(a, dtype=np.float64).ravel()).to(ctx.device)


def periodic_patches(m):
    """the x-min and x-max wall faces of a hex box as a cyclic patch pair (neighbRank -(partner + 1))"""
    nx, ny, nz = m.nx, m.ny, m.nz
    jk = np.arange(ny * nz)
    lo, hi = jk * nx, jk * nx + nx - 1
    return np.array([0, ny * nz, 2 * ny * nz], np.int32), np.concatenate([lo, hi]).astype(np.int32)


class Case:
    """one hex mesh with a boundary list, its symmetric (pressure) and asymmetric (momentum) fvMatrix, and a GAMG
    hierarchy on the symmetric one"""

    def __init__(self, gpu, meshmod, orc, gamg=False):
        capi, ctx, torch = gpu
        self.capi, self.torch = capi, torch
        self.t = lambda a: tensor(ctx, torch, a)
        m, _, self.p = poisson_case(meshmod, orc, DIMS)
        _, _, self.u = momentum_case(meshmod, orc, DIMS)
        self.m = m
        self.addr = capi.mesh_to_device(ctx, m)
        capi.fv_boundary_set(self.addr, self.p["bfc"])
        self.P, self.U = capi.LduMatrix(self.addr), capi.LduMatrix(self.addr)
        self.set()
        self.fvP = self.fv(self.P, self.p, 1)
        self.fvU = self.fv(self.U, self.u, 3)
        self.gg = capi.GamgAgglomeration(self.addr, meshmod.face_area_pair_weights(m), 10) if gamg else None

    def fv(self, mat, d, nc):
        psi = np.random.default_rng(nc).uniform(-1, 1, (self.m.nCells, nc))
        return self.capi.FvMatrix(mat, nc, self.t(d["diag"]), self.t(d["source"]), self.t(psi), self.t(d["V"]),
                                  self.t(d["ic"]), self.t(d["bc"]))

    def set(self):
        self.P.set(self.t(self.p["diag"]), self.t(self.p["upper"]))
        self.U.set(self.t(self.u["diag"]), self.t(self.u["upper"]), self.t(self.u["lower"]))

    def close(self):
        if self.gg is not None:
            self.gg.close()
        self.P.close()
        self.U.close()
        self.addr.close()


def _symmetric(gpu, meshmod, orc):
    c = Case(gpu, meshmod, orc)
    assert c.addr.info()["faceStream"]
    psi, b = c.t(np.zeros(c.m.nCells)), c.t(c.p["source"])
    c.P.solve("PCG", "DIC", psi, b, histCap=32, maxIter=20)
    c.P.Amul(psi), c.P.residual(psi, b)
    return [c]


def _asymmetric(gpu, meshmod, orc):
    c = Case(gpu, meshmod, orc)
    psi, b = c.t(np.zeros(c.m.nCells)), c.t(c.u["source"][:, 0])
    c.U.solve("PBiCG", "DILU", psi, b, histCap=32, maxIter=20)
    c.U.Tmul(psi)
    return [c]


def _cyclic(gpu, meshmod, orc):
    capi, ctx, torch = gpu
    m = meshmod.hex_mesh(*DIMS)
    ps, fc = periodic_patches(m)
    addr = capi.LduAddressing(ctx, m.nCells, m.lower, m.upper, ps, fc, np.array([-2, -1], np.int32), m.cell_centres())
    c = meshmod.pressure_laplacian(m)
    t = lambda a: tensor(ctx, torch, a)
    ifc = t(np.full(len(fc), -0.1))
    mat = capi.LduMatrix(addr).set(t(c["diag"]), t(c["upper"]), None, ifc, ifc)
    psi = t(np.zeros(m.nCells))
    mat.solve("PCG", "DIC", psi, t(np.ones(m.nCells)), maxIter=20)
    mat.Amul(psi)
    return [mat, addr]


def _boundary_twice(gpu, meshmod, orc):
    c = Case(gpu, meshmod, orc)
    bfc = np.asarray(c.p["bfc"])
    c.capi.fv_boundary_set(c.addr, bfc[: len(bfc) // 3])
    c.capi.fv_boundary_set(c.addr, np.concatenate([bfc, bfc[:7]]))
    return [c]


def _fvm(nc):
    def run(gpu, meshmod, orc):
        c = Case(gpu, meshmod, orc)
        fv = c.fvP if nc == 1 else c.fvU
        fv.A(), fv.H(), fv.flux(len(c.p["bfc"])), fv.residual()
        fv.solve("PCG" if nc == 1 else "PBiCG", "DIC" if nc == 1 else "DILU", maxIter=20)
        return [c]
    return run


def _mules(gpu, meshmod, orc):
    capi, ctx, torch = gpu
    d = mules_case(meshmod, DIMS, seed=12)
    addr = capi.mesh_to_device(ctx, d["m"])
    capi.fv_boundary_set(addr, d["bfc"])
    t = lambda a: tensor(ctx, torch, a)
    capi.mules_limiter(addr, t(d["V"]), d["rDeltaT"], t(d["psi"]), t(d["psi0"]), t(d["psiB"]), t(d["phi"]), t(d["phiB"]),
                       t(d["phiPsi"]), t(d["phiPsiB"]), 1.0, 0.0, 3)
    return [addr]


def _gamg(direct):
    def run(gpu, meshmod, orc):
        c = Case(gpu, meshmod, orc, gamg=True)
        psi, b = c.t(np.zeros(c.m.nCells)), c.t(c.p["source"])
        perf, _ = c.P.solve("GAMG", "GaussSeidel", psi, b, gamg=c.gg, histCap=32, tolerance=1e-8, maxIter=30,
                            directSolveCoarsest=direct)
        assert perf.nIterations > 0
        return [c]
    return run


ROUND_TRIPS = {"symmetric-face-stream": _symmetric, "asymmetric": _asymmetric, "cyclic": _cyclic,
               "boundary-set-twice": _boundary_twice, "fvm-nComp1": _fvm(1), "fvm-nComp3": _fvm(3), "mules": _mules,
               "gamg-direct": _gamg(1), "gamg-iterative": _gamg(0)}


@pytest.mark.parametrize("name", list(ROUND_TRIPS))
def test_handles_give_back_their_memory(gpu, meshmod, orc, name):
    capi, ctx, torch = gpu
    live0, n0 = device_mem(capi, ctx)
    handles = ROUND_TRIPS[name](gpu, meshmod, orc)
    ctx.sync()
    live1, n1 = device_mem(capi, ctx)
    assert live1 > live0 and n1 > n0
    for h in handles:
        h.close()
    assert device_mem(capi, ctx)[0] == live0


def test_failed_create_leaves_nothing(gpu, meshmod):
    """an unmatched cyclic partner is found after the layout was uploaded"""
    capi, ctx, torch = gpu
    m = meshmod.hex_mesh(*DIMS)
    ps, fc = periodic_patches(m)
    live0, n0 = device_mem(capi, ctx)
    with pytest.raises(capi.B200LduError) as e:
        capi.LduAddressing(ctx, m.nCells, m.lower, m.upper, ps, fc, np.array([-2, -2], np.int32), m.cell_centres())
    assert e.value.rc == -1 and b"no matching partner" in capi.lib().b200ldu_last_error()
    live1, n1 = device_mem(capi, ctx)
    assert n1 > n0, "the layout should have been uploaded before the partner check"
    assert live1 == live0


def test_steady_state_allocates_nothing(gpu, meshmod, orc):
    capi, ctx, torch = gpu
    c = Case(gpu, meshmod, orc, gamg=True)
    t, n = c.t, c.m.nCells
    d = mules_case(meshmod, DIMS, seed=12)
    assert np.array_equal(d["bfc"], c.p["bfc"])
    mules_args = [t(d[k]) for k in ("V",)] + [d["rDeltaT"]] + [t(d[k]) for k in ("psi", "psi0", "psiB", "phi", "phiB",
                                                                               "phiPsi", "phiPsiB")]
    x, b, bu = t(np.random.default_rng(1).uniform(-1, 1, n)), t(c.p["source"]), t(c.u["source"][:, 0])

    def sequence():
        c.set()
        c.P.solve("PCG", "DIC", x.clone(), b, histCap=64, maxIter=20)
        c.P.solve("GAMG", "GaussSeidel", x.clone(), b, gamg=c.gg, maxIter=5)
        c.U.solve("PBiCG", "DILU", x.clone(), bu, maxIter=20)
        c.fvU.solve("PBiCG", "DILU", maxIter=20)
        c.fvP.residual()
        capi.mules_limiter(c.addr, *mules_args, 1.0, 0.0, 3)
        c.P.Amul(x), c.P.residual(x, b), c.P.precondition("DIC", x), c.P.smooth("GaussSeidel", x, b, 2)
        ctx.sync()

    sequence()
    warm = device_mem(capi, ctx)
    for _ in range(3):
        sequence()
        assert device_mem(capi, ctx) == warm
    c.close()


def test_stream_switch_keeps_one_stream(gpu, meshmod, orc):
    capi, ctx, torch = gpu
    c = Case(gpu, meshmod, orc)
    assert c.addr.info()["faceStream"]
    diag, upper, lower = c.t(c.p["diag"]), c.t(c.p["upper"]), c.t(c.u["lower"])
    c.P.set(diag, upper)
    live_sym = device_mem(capi, ctx)[0]
    c.P.set(diag, upper, lower)
    assert device_mem(capi, ctx)[0] != live_sym
    c.P.set(diag, upper)
    assert device_mem(capi, ctx)[0] == live_sym
    c.close()
