"""The face stream's template table: the column and product-slot words of every slice's owner block and every band's
list are stored once per distinct block, and each slice and band refers to its block.  Without a GPU: the table is
exactly the blocks its slices and bands refer to, it does not depend on the number of threads that built it, it stays
small on structured meshes, and the words it stands for (layout code 11) pass the face stream's structural check
also where nothing repeats.  On the GPU: such a mesh gives the entry stream's results bit for bit."""
import ctypes as C
import importlib

import numpy as np
import pytest
from layout_helpers import debug_addr, debug_layout, debug_lib
from test_face_stream_cpu import _check_structure

# b200ldu_layout_debug_get codes (layout.cu)
CODES = {"fsSlice": (10, np.int32), "fsCT": (11, np.uint32), "fsListStart": (13, np.int32), "fsDims": (15, np.int64),
         "fsTpl": (16, np.uint32), "tpl64": (17, np.int32), "fsListTpl": (18, np.int32)}


@pytest.fixture(scope="module")
def capi():
    g = importlib.import_module("__graft_entry__")
    g.build()
    return importlib.import_module("rapidcfd-dev_b200.capi")


def _templates(capi, mesh, centres=True, band=None, words=False):
    """{name: array} of the face-stream arrays in CODES (the expanded words only when `words`)"""
    L = debug_lib(capi)
    h = debug_addr(capi, mesh, centres, band)
    out = {}
    for name, (what, dt) in CODES.items():
        if name == "fsCT" and not words:
            continue
        n = L.b200ldu_layout_debug_get(h, what, None, 0)
        a = np.zeros(max(n, 1), dtype=dt)
        L.b200ldu_layout_debug_get(h, what, a.ctypes.data, n)
        out[name] = a[:n]
    L.b200ldu_layout_debug_destroy(h)
    return out


def _blocks(t):
    """(offset, words) of the block every slice, then every band, refers to"""
    wo = (t["fsSlice"].reshape(-1, 4)[:, 2] & 0xFFFF).astype(np.int64)
    own = np.stack([t["tpl64"].astype(np.int64) * 64, wo * 64], 1)
    ls = t["fsListStart"].astype(np.int64)
    lst = np.stack([t["fsListTpl"].astype(np.int64), np.diff(ls)], 1)
    return own, lst


def _check_table(t):
    """every offset in range, owner blocks wo x 64 words at multiples of 64, and the distinct blocks tile the table
    exactly: every template is referenced and no word is stored twice; returns the number of templates"""
    own, lst = _blocks(t)
    size = len(t["fsTpl"])
    both = np.concatenate([own, lst])
    assert np.all(both[:, 0] >= 0) and np.all(both[:, 1] >= 0) and np.all(both.sum(1) <= size)
    assert np.all(own[:, 0] % 64 == 0)
    pos = 0
    distinct = sorted(set(map(tuple, both.tolist())))
    for off, n in distinct:
        assert off == pos, (off, pos)
        pos += n
    assert pos == size
    return len(distinct)


def _expand(t):
    """the words of every face-stream entry, gathered from the table"""
    own, lst = _blocks(t)
    start = t["fsSlice"].reshape(-1, 4)[:, 0].astype(np.int64) * 64
    ls = t["fsListStart"].astype(np.int64)
    ct = np.zeros(int(ls[-1]), np.uint32)
    for s, (off, n) in enumerate(own):
        ct[start[s]:start[s] + n] = t["fsTpl"][off:off + n]
    for b, (off, n) in enumerate(lst):
        ct[ls[b]:ls[b] + n] = t["fsTpl"][off:off + n]
    return ct


@pytest.mark.parametrize("dims,centres,band", [((16, 16, 16), True, 512), ((12, 12, 12), False, 256),
                                               ((7, 3, 5), False, None)])
def test_table_invariants(capi, meshmod, dims, centres, band):
    mesh = meshmod.hex_mesh(*dims)
    t = _templates(capi, mesh, centres, band, words=True)
    _check_table(t)
    assert np.array_equal(_expand(t), t["fsCT"])


def test_table_with_processor_patches(capi, meshmod):
    for rank in range(4):
        mesh = meshmod.decompose(8, 4, rank)
        t = _templates(capi, mesh, True, 64, words=True)
        _check_table(t)
        assert np.array_equal(_expand(t), t["fsCT"])


def test_table_is_deterministic(capi, meshmod):
    """two builds, and builds on 1, 3 and the default number of OpenMP threads, give the same table"""
    gomp = C.CDLL("libgomp.so.1")
    default = gomp.omp_get_max_threads()
    mesh = meshmod.hex_mesh(40, 36, 32)
    keys = ("fsTpl", "tpl64", "fsListTpl")
    runs = []
    try:
        for nt in (default, default, 1, 3):
            gomp.omp_set_num_threads(nt)
            t = _templates(capi, mesh, False, 512)
            runs.append([t[k] for k in keys])
    finally:
        gomp.omp_set_num_threads(default)
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("case", ["hex128", "rank0_of_2x2x2_256"])
def test_table_is_small_on_structured_meshes(capi, meshmod, case):
    """at the band size the library picks, the distinct blocks stay under 1 % of the slices"""
    mesh = meshmod.hex_mesh(128) if case == "hex128" else meshmod.decompose(256, 8, 0)
    t = _templates(capi, mesh)
    n = _check_table(t)
    nSlices = len(t["tpl64"])
    print(f"\n[templates] {case}: {n} templates for {nSlices} slices and {len(t['fsListTpl'])} bands, "
          f"{len(t['fsTpl'])} words against {int(t['fsDims'][0] + t['fsDims'][1])} entries")
    assert n < 0.01 * nSlices


class _Renumbered:
    """An n-cell hex mesh with its cells numbered at random and no cell centres: slices and bands rarely repeat."""

    def __init__(self, meshmod, dims, seed):
        m = meshmod.hex_mesh(*dims)
        p = np.random.default_rng(seed).permutation(m.nCells)  # new number of each cell
        a, b = p[np.asarray(m.lower)], p[np.asarray(m.upper)]
        lo, hi = np.minimum(a, b), np.maximum(a, b)
        order = np.lexsort((hi, lo))
        self.lower, self.upper = lo[order].astype(np.int32), hi[order].astype(np.int32)
        self.nCells, self.nFaces = m.nCells, len(order)

    def cell_centres(self):
        return None

    def patch_start_facecells(self):
        return np.zeros(1, np.int32), np.zeros(0, np.int32)


def test_renumbered_mesh_without_centres(capi, meshmod):
    mesh = _Renumbered(meshmod, (16, 12, 10), 7)
    lay = debug_layout(capi, mesh, centres=False, band=256)
    _check_structure(mesh, lay)
    t = _templates(capi, mesh, False, 256, words=True)
    _check_table(t)
    assert np.array_equal(_expand(t), lay["fsCT"])


@pytest.mark.gpu
def test_renumbered_mesh_streams_agree(meshmod, orc):
    """Amul and PCG on the face stream, which reads its words from the table, bit for bit the entry stream's"""
    import torch
    from test_gpu_engine_streams import Mismatches, Problem, Side, _same_solve, _solve
    assert torch.cuda.is_available()
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    mesh = _Renumbered(meshmod, (40, 24, 20), 11)
    rng = np.random.default_rng(13)
    up = rng.uniform(-1.0, 1.0, mesh.nFaces)
    s = np.zeros(mesh.nCells)
    np.add.at(s, mesh.lower, np.abs(up))
    np.add.at(s, mesh.upper, np.abs(up))
    diag = -(s + 0.1) * rng.uniform(1.0, 1.5, mesh.nCells)
    pb = Problem(orc, mesh.nCells, mesh.lower, mesh.upper, diag, up, seed=5)
    ctx = capi.Context(0)
    gpu = (capi, ctx, torch)
    es, fs = Side(gpu, pb, 512, 0), Side(gpu, pb, 512, 1)
    try:
        assert fs.info["faceStream"] and not es.info["faceStream"], fs.info
        assert fs.info["fsTemplateWords"] > 0 and fs.info["fsTemplates"] > 0, fs.info
        M = Mismatches()
        for seed in (3, 4):
            x = pb.field(seed)
            a_es, a_fs = (side.mat.Amul(side.t(x)).cpu().numpy() for side in (es, fs))
            M.bits_es(a_es, a_fs, f"Amul [{seed}] ES vs FS")
            M.bits(a_fs, pb.om.amul(x), f"Amul [{seed}] FS vs oracle")
        b = pb.om.amul(pb.field(42))
        for ctl in (dict(tolerance=0.0, maxIter=25), dict(tolerance=1e-8, maxIter=1000)):
            _same_solve(M, _solve(es, "PCG", "DIC", b, **ctl), _solve(fs, "PCG", "DIC", b, **ctl), f"PCG DIC {ctl}")
        M.check()
    finally:
        es.close()
        fs.close()
        ctx.close()
