"""The fused PCG adds each body's alpha p to psi in the next body's second sweep, and closes the solve with one
residual-only step and at most one deferred psi update.  Whatever the host's chunking (checkEvery) and whether
chunks are replayed as CUDA graphs, psi, the residual history and the iteration count must be the same bits, and
follow the oracle -- also when the last body ends on a chunk boundary, the solve stops mid-chunk, or it never
iterates."""
import importlib
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


def mid_chunk_tolerance(href):
    """A tolerance the residual history first falls below at an iteration k past the first chunk of 8 bodies (the
    second is replayed from a graph) that is no multiple of 5 or 8, with a 0.1 % margin on both sides."""
    for k in range(9, len(href)):
        if k % 5 and k % 8 and href[k] < 0.999 * href[:k].min():
            return float(np.sqrt(href[k] * href[:k].min())), k
    raise AssertionError("no residual drop to converge on")


@pytest.mark.parametrize("pre", ["DIC", "diagonal", "none"])
@pytest.mark.parametrize("dims", [(18, 14, 10), (32, 32, 32)])
def test_close_independent_of_chunking(gpu, meshmod, orc, pre, dims):
    capi, ctx, torch = gpu
    m = meshmod.hex_mesh(*dims)
    c = meshmod.pressure_laplacian(m)
    oa = orc.Addr(m.nCells, m.lower, m.upper)
    om = orc.Matrix(oa, c["diag"], c["upper"], None)
    b = om.amul(meshmod.cell_field_global(m, 42))
    psi0 = 0.1 * meshmod.cell_field_global(m, 7)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(ctx.device)
    addr = capi.mesh_to_device(ctx, m)
    mat = capi.LduMatrix(addr)
    mat.set(t(c["diag"]), t(c["upper"]))
    bd = t(b)

    _, _, hfull = om.solve("PCG", pre, psi0, b, tolerance=0.0, maxIter=40)
    tol, kConv = mid_chunk_tolerance(hfull)
    cases = {
        "converges mid-chunk": dict(tolerance=tol, maxIter=100),
        "maxIter 14": dict(tolerance=0.0, maxIter=14),
        "maxIter 15": dict(tolerance=0.0, maxIter=15),
        "maxIter 16": dict(tolerance=0.0, maxIter=16),
        "maxIter 0": dict(tolerance=0.0, maxIter=0),
        "minIter > maxIter + 1": dict(tolerance=0.0, maxIter=3, minIter=7),
        "converged at the initial residual": dict(tolerance=1e30, maxIter=50),
    }
    saved = {k: os.environ.get(k) for k in ("B200LDU_GRAPH", "B200LDU_PCG_FUSED")}
    os.environ.pop("B200LDU_PCG_FUSED", None)
    try:
        for name, ctl in cases.items():
            psi_ref, pr, href = om.solve("PCG", pre, psi0, b, **ctl)
            runs = []
            for graph in ("0", "1"):
                os.environ["B200LDU_GRAPH"] = graph
                for every in (1, 5, 8):
                    psi = t(psi0)
                    perf, hist = mat.solve("PCG", pre, psi, bd, histCap=512, checkEvery=every, **ctl)
                    runs.append(((graph, every), perf.nIterations, perf.converged, hist.copy(), psi.cpu().numpy()))
            _, n0, conv0, h0, x0 = runs[0]
            for key, n, conv, h, x in runs[1:]:
                assert n == n0 and conv == conv0, (name, key)
                assert np.array_equal(h, h0), (name, key)
                assert np.array_equal(x, x0), (name, key)
            assert n0 == pr.nIterations, (name, n0, pr.nIterations)
            assert conv0 == pr.converged, name
            assert len(h0) == n0 + 1, name
            k = min(30, len(h0), len(href))
            np.testing.assert_allclose(h0[:k], href[:k], rtol=1e-9, err_msg=name)
            np.testing.assert_allclose(x0, psi_ref, rtol=0, atol=2e-7, err_msg=name)
            if name == "converges mid-chunk":
                assert n0 == kConv
            if name == "maxIter 0":
                assert n0 == 1
            if name == "minIter > maxIter + 1":
                assert n0 == 7
            if name == "converged at the initial residual":
                assert n0 == 0 and np.array_equal(x0, psi0)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    mat.close()
    addr.close()
