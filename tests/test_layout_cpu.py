"""Host logic of the product library without a GPU: the C-ABI library loads and exports
every symbol include/b200ldu.h declares, and the banded layout (renumbering + slot-major
entries + halo lists) is structurally exact: reassembling the entries through the
permutation reproduces the LDU matrix pattern face for face, in the reference's row order."""
import ctypes as C
import importlib
import os
import re

import numpy as np
import pytest
from layout_helpers import debug_layout, debug_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def capi():
    g = importlib.import_module("__graft_entry__")
    g.build()
    return importlib.import_module("rapidcfd-dev_b200.capi")


def test_library_exports_header_symbols(capi):
    hdr = open(os.path.join(ROOT, "include", "b200ldu.h")).read()
    names = sorted(set(re.findall(r"\b(b200ldu_[a-z0-9_A-Z]+)\s*\(", hdr)))
    assert len(names) >= 40
    L = capi.lib()
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing
    assert set(capi.EXPORTS) <= set(names)


def test_no_gpu_is_a_loud_error(capi):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = C.c_void_p()
    rc = capi.lib().b200ldu_ctx_create(0, C.byref(h))
    assert rc == -2
    assert b"no CPU fallback" in capi.lib().b200ldu_last_error()
    with pytest.raises(RuntimeError):
        capi.Context(0)


def _check_layout(mesh, lay):
    nPad, nBands, bandRows, nRecv, maxHalo = [int(x) for x in lay["dims"]]
    n = mesh.nCells
    perm, iperm = lay["perm"], lay["iperm"]
    assert sorted(perm.tolist()) == list(range(n))
    assert np.array_equal(iperm[perm], np.arange(n)) and np.all(iperm[n:] == -1)
    assert nPad % bandRows == 0 and bandRows % 64 == 0 and nBands * bandRows == nPad
    # reference row order per cell: owner faces, then losort (ascending face), then interfaces
    own = [[] for _ in range(n)]
    nei = [[] for _ in range(n)]
    for f in range(mesh.nFaces):
        own[mesh.lower[f]].append(f)
        nei[mesh.upper[f]].append(f)
    ps, fc = mesh.patch_start_facecells()
    ifc = [[] for _ in range(n)]
    for i, c in enumerate(fc):
        ifc[c].append(i)
    nSlices = nPad // 64
    seen_codes = []
    for s in range(nSlices):
        base, W, WL = int(lay["sliceStart"][s]), int(lay["sliceW"][s]), int(lay["sliceWL"][s])
        band = (s * 64) // bandRows
        hs = lay["haloStart"][band]
        halo = lay["haloIdx"][hs:lay["haloStart"][band + 1]]
        assert np.all(np.diff(halo) > 0)
        assert len(halo) <= maxHalo
        for q in range(64):
            r = s * 64 + q
            c = iperm[r]
            cols = lay["col"][base + q: base + 64 * W: 64] if W else np.zeros(0, np.uint16)
            codes = lay["code"][base + q: base + 64 * W: 64] if W else np.zeros(0, np.int32)

            def target(cv):
                return band * bandRows + cv if cv < bandRows else int(halo[cv - bandRows])
            if c < 0:
                assert np.all(codes == -1)
                continue
            exp = [(2 * f, perm[mesh.upper[f]]) for f in own[c]] + [(2 * f + 1, perm[mesh.lower[f]]) for f in nei[c]]
            assert len(exp) <= WL
            got_local = [(int(codes[j]), target(int(cols[j]))) for j in range(WL) if codes[j] != -1]
            assert got_local == [(a, int(b)) for a, b in exp]
            # padding slots point at the row itself with a zero coefficient
            for j in range(W):
                if codes[j] == -1:
                    assert target(int(cols[j])) == r
            got_if = [(int(codes[j]), target(int(cols[j]))) for j in range(WL, W) if codes[j] != -1]
            assert got_if == [(-2 - i, nPad + i) for i in ifc[c]]
            seen_codes += [int(x) for x in codes if x != -1]
    assert sorted(x for x in seen_codes if x >= 0) == list(range(2 * mesh.nFaces))
    assert sorted(-2 - x for x in seen_codes if x < -1) == list(range(nRecv))


@pytest.mark.parametrize("dims,centres,band", [((6, 5, 4), True, None), ((8, 8, 8), True, 128),
                                               ((7, 3, 5), False, None), ((12, 12, 12), False, 256),
                                               ((1, 1, 1), True, None), ((5, 1, 1), True, None)])
def test_layout_structure(capi, meshmod, dims, centres, band):
    mesh = meshmod.hex_mesh(*dims)
    _check_layout(mesh, debug_layout(capi, mesh, centres, band))


def test_layout_with_processor_patches(capi, meshmod):
    for rank in range(4):
        mesh = meshmod.decompose(8, 4, rank)
        lay = debug_layout(capi, mesh, True, 64)
        assert lay["dims"][3] == sum(len(p.faceCells) for p in mesh.coupled_patches()) > 0
        _check_layout(mesh, lay)


def test_layout_bricks_are_compact(capi, meshmod):
    """32^3 with 512-row bands: Morton tiles of 8x8x8 => every band is one brick and its halo is
    exactly the brick's face-adjacent cells (<= 6*64)."""
    mesh = meshmod.hex_mesh(32)
    lay = debug_layout(capi, mesh, True, 512)
    nPad, nBands, bandRows, nRecv, maxHalo = [int(x) for x in lay["dims"]]
    assert bandRows == 512 and nBands == 64
    assert maxHalo <= 6 * 64
    cc = mesh.cell_centres()
    iperm = lay["iperm"]
    for b in range(nBands):
        cells = iperm[b * 512:(b + 1) * 512]
        ext = cc[cells].max(0) - cc[cells].min(0)
        assert np.allclose(ext, 7 * mesh.h)


def test_layout_rejects_bad_addressing(capi):
    L = debug_lib(capi)
    l = np.array([1, 0], np.int32)  # not owner-sorted
    u = np.array([2, 1], np.int32)
    h = C.c_void_p()
    rc = L.b200ldu_layout_debug_create(3, 2, l.ctypes.data, u.ctypes.data, 0, None, None, None, C.byref(h))
    assert rc == -1


class _RandomGraph:
    """LDU pattern of a random graph without any locality (worst case for the band tiles)."""

    def __init__(self, n, k, seed):
        rng = np.random.default_rng(seed)
        a, b = rng.integers(0, n, size=n * k), rng.integers(0, n, size=n * k)
        keep = a != b
        pr = np.unique(np.stack([np.minimum(a, b)[keep], np.maximum(a, b)[keep]], 1), axis=0).astype(np.int32)
        self.lower, self.upper = pr[:, 0].copy(), pr[:, 1].copy()
        self.nCells, self.nFaces = n, len(pr)

    def cell_centres(self):
        return None

    def patch_start_facecells(self):
        return np.zeros(1, np.int32), np.zeros(0, np.int32)


def test_layout_narrows_bands_until_the_tile_fits(capi):
    """A band's rows + halo columns are staged in shared memory (the check allows for two vectors): when a
    numbering without locality makes that tile too large -- or needs more than 65535 columns -- the
    builder halves bandRows until it fits instead of failing at launch time."""
    g = _RandomGraph(30000, 6, 1)
    lay = debug_layout(capi, g, centres=False, band=16384)
    nPad, nBands, bandRows, nRecv, maxHalo = [int(x) for x in lay["dims"]]
    assert bandRows < 16384 and (bandRows + maxHalo + 2) * 16 <= 200 * 1024
    _check_layout(g, lay)
