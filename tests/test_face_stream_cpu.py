"""Face stream of symmetric matrices without a GPU: every face is stored once in its owner's row, every product
for a neighbour row has exactly one slot in its band's shared-memory buffer, and a scalar replay of the engine's
two passes (owner pass + list, then each row's buffer slots in order) reproduces the oracle's Amul bit for bit."""
import importlib

import numpy as np
import pytest
from layout_helpers import debug_layout

FS_PAD, FS_NONE = 0xFFFE, 0xFFFF


@pytest.fixture(scope="module")
def capi():
    g = importlib.import_module("__graft_entry__")
    g.build()
    return importlib.import_module("rapidcfd-dev_b200.capi")


class _Fs:
    """The face stream of one layout, decoded."""

    def __init__(self, lay):
        self.nPad, self.nBands, self.bandRows, self.nRecv, self.maxHalo = [int(x) for x in lay["dims"]]
        self.nOwn, self.nList, self.bufMax, self.used = [int(x) for x in lay["fsDims"]]
        assert len(lay["fsCT"]) == self.nOwn + self.nList
        sl = lay["fsSlice"].reshape(-1, 4)
        assert len(sl) == self.nPad // 64
        self.start = sl[:, 0].astype(np.int64) * 64
        self.bufOff = sl[:, 1]
        self.wo, self.wn, self.wi = sl[:, 2] & 0xFFFF, sl[:, 2] >> 16, sl[:, 3]
        self.ct, self.code = lay["fsCT"], lay["fsCode"]
        self.col, self.slot = (self.ct & 0xFFFF).astype(np.int64), (self.ct >> 16).astype(np.int64)
        self.ls, self.li = lay["fsListStart"], lay["fsListIfc"]
        self.haloStart, self.haloIdx = lay["haloStart"], lay["haloIdx"]
        self.spb = self.bandRows // 64

    def target(self, band, cols):
        """extended index (banded row, or nPad + received slot) of tile columns of `band`"""
        cols = np.asarray(cols, np.int64)
        own = cols < self.bandRows
        hidx = np.where(own, 0, cols - self.bandRows) + self.haloStart[band]
        return np.where(own, band * self.bandRows + cols, self.haloIdx[np.minimum(hidx, len(self.haloIdx) - 1)])

    def owner_entries(self, s):
        """(entry indices [wo, 64]) of slice s"""
        return self.start[s] + np.arange(int(self.wo[s]))[:, None] * 64 + np.arange(64)[None, :]

    def slot_of(self, row, j):
        s = row // 64
        return int(self.bufOff[s]) + j * 64 + row % 64


def _check_structure(mesh, lay, patches=None):
    fs = _Fs(lay)
    perm, iperm = lay["perm"], lay["iperm"]
    ps, fc = patches if patches is not None else mesh.patch_start_facecells()
    lower, upper = np.asarray(mesh.lower), np.asarray(mesh.upper)
    band = lambda r: int(r) // fs.bandRows
    # losort position of every face at its neighbour cell
    nb = np.zeros(mesh.nFaces, np.int64)
    cnt = np.zeros(mesh.nCells, np.int64)
    for f in range(mesh.nFaces):
        nb[f] = cnt[upper[f]]
        cnt[upper[f]] += 1
    ifc_pos = {}
    seen = {}
    for i, c in enumerate(fc):
        ifc_pos[i] = seen.get(int(c), 0)
        seen[int(c)] = ifc_pos[i] + 1
    owner_faces = []
    slots = [[] for _ in range(fs.nBands)]
    for s in range(fs.nPad // 64):
        b = s * 64 // fs.bandRows
        e = fs.owner_entries(s)
        for q in range(64):
            r = s * 64 + q
            codes, t, cols = fs.code[e[:, q]], fs.slot[e[:, q]], fs.col[e[:, q]]
            pad = t == FS_PAD
            assert np.all(codes[pad] == -1) and np.all(codes[~pad] >= 0) and np.all(codes[~pad] % 2 == 0)
            assert np.all(pad[np.argmax(pad):]) if pad.any() else True  # padding at the end
            c = iperm[r]
            fo = codes[~pad] // 2
            assert list(fo) == (sorted(fo) if c >= 0 else [])
            if c >= 0:
                assert np.all(lower[fo] == c)
            owner_faces += list(fo)
            for f, tt, cv in zip(fo, t[~pad], cols[~pad]):
                n = perm[upper[f]]
                assert fs.target(b, [cv])[0] == n
                if band(n) == b:
                    assert tt == fs.slot_of(n, 1 + nb[f])
                    slots[b].append(int(tt))
                else:
                    assert tt == FS_NONE
    # every face exactly once as an owner entry
    assert sorted(owner_faces) == list(range(mesh.nFaces))
    # lists: every cross-band neighbour side and every interface face exactly once
    assert fs.ls[0] == fs.nOwn and fs.ls[-1] == fs.nOwn + fs.nList
    got_x, got_i = [], []
    for b in range(fs.nBands):
        assert fs.ls[b] <= fs.li[b] <= fs.ls[b + 1]
        for i in range(fs.ls[b], fs.li[b]):
            f = fs.code[i] // 2
            assert fs.code[i] % 2 == 1
            n, o = perm[upper[f]], perm[lower[f]]
            assert band(n) == b and band(o) != b and fs.target(b, [fs.col[i]])[0] == o
            assert fs.slot[i] == fs.slot_of(n, 1 + nb[f])
            got_x.append(int(f))
            slots[b].append(int(fs.slot[i]))
        for i in range(fs.li[b], fs.ls[b + 1]):
            pf = -2 - fs.code[i]
            n = perm[fc[pf]]
            assert band(n) == b and fs.target(b, [fs.col[i]])[0] == fs.nPad + pf
            assert fs.slot[i] == fs.slot_of(n, 1 + int(fs.wn[n // 64]) + ifc_pos[pf])
            got_i.append(int(pf))
            slots[b].append(int(fs.slot[i]))
    cross = [f for f in range(mesh.nFaces) if band(perm[upper[f]]) != band(perm[lower[f]])]
    assert sorted(got_x) == cross
    assert sorted(got_i) == list(range(len(fc)))
    # no two products share a slot, none lands on a row's owner-pass sum (slot 0), all fit the buffer
    for b in range(fs.nBands):
        sb = np.array(slots[b], np.int64)
        assert len(np.unique(sb)) == len(sb)
        s0 = {int(fs.bufOff[s]) + q for s in range(b * fs.spb, (b + 1) * fs.spb) for q in range(64)}
        assert not (set(sb.tolist()) & s0)
        assert np.all(sb < fs.bufMax)
    return fs


def _replay_amul(lay, diag, upper, bou, psi, recv):
    """Scalar replay of engine_kernel<AmulOp, FS> on the host, same operations in the same order."""
    fs = _Fs(lay)
    perm = lay["perm"]
    xb = np.zeros(fs.nPad + fs.nRecv)
    xb[perm] = psi
    xb[fs.nPad:] = recv
    dg = np.ones(fs.nPad)
    dg[perm] = diag
    code = fs.code
    val = np.where(code >= 0, upper[np.maximum(code, 0) // 2], 0.0)
    ifc = code < -1
    val[ifc] = -np.asarray(bou)[-2 - code[ifc]]
    acc = dg * xb[:fs.nPad]
    buf = np.full((fs.nBands, max(fs.bufMax, 1)), -0.0)
    for s in range(fs.nPad // 64):
        b = s * 64 // fs.bandRows
        rows = s * 64 + np.arange(64)
        for j in range(int(fs.wo[s])):
            e = fs.start[s] + j * 64 + np.arange(64)
            t, v, g = fs.slot[e], val[e], fs.target(b, fs.col[e])
            real = t != FS_PAD
            acc[rows[real]] = acc[rows[real]] + v[real] * xb[g[real]]
            st = t < FS_PAD
            buf[b, t[st]] = v[st] * xb[rows[st]]
        buf[b, int(fs.bufOff[s]) + np.arange(64)] = acc[rows]
    for b in range(fs.nBands):
        i = np.arange(fs.ls[b], fs.ls[b + 1])
        buf[b, fs.slot[i]] = val[i] * xb[fs.target(b, fs.col[i])]
    out = np.empty(fs.nPad)
    for s in range(fs.nPad // 64):
        b = s * 64 // fs.bandRows
        base = int(fs.bufOff[s]) + np.arange(64)
        a = buf[b, base]
        for j in range(1, 1 + int(fs.wn[s]) + int(fs.wi[s])):
            a = a + buf[b, base + j * 64]
        out[s * 64:(s + 1) * 64] = a
    return out[perm]


def _bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.int64)


def _check_replay(orc, meshmod, mesh, lay, coef, patches=None, neighbRank=None, comm_recv=None):
    ps, fc = patches if patches is not None else mesh.patch_start_facecells()
    a = orc.Addr(mesh.nCells, mesh.lower, mesh.upper, ps if len(fc) else None, fc if len(fc) else None,
                 neighbRank=neighbRank)
    m = orc.Matrix(a, coef["diag"], coef["upper"], None, coef.get("bou"), coef.get("bou"))
    psi = meshmod.cell_field_global(mesh, 11)
    comm = None
    if comm_recv is not None:
        comm = orc.PyComm(halo=lambda send, starts: comm_recv.copy())
    ref = m.amul(psi, comm)
    recv = a.patch_neighbour_field(psi, comm) if len(fc) else np.zeros(0)
    bou = coef.get("bou") if coef.get("bou") is not None else np.zeros(0)
    got = _replay_amul(lay, coef["diag"], coef["upper"], bou, psi, recv)
    assert np.array_equal(_bits(got), _bits(ref))


@pytest.mark.parametrize("dims,centres,band", [((6, 5, 4), True, None), ((8, 8, 8), True, 128),
                                               ((7, 3, 5), False, None), ((12, 12, 12), False, 256),
                                               ((16, 16, 16), True, 512), ((1, 1, 1), True, None)])
def test_face_stream_hex(capi, orc, meshmod, dims, centres, band):
    mesh = meshmod.hex_mesh(*dims)
    lay = debug_layout(capi, mesh, centres, band)
    _check_structure(mesh, lay)
    coef = meshmod.pressure_laplacian(mesh)
    _check_replay(orc, meshmod, mesh, lay, dict(diag=coef["diag"], upper=coef["upper"]))


def test_face_stream_processor_patches(capi, orc, meshmod):
    for rank in range(4):
        mesh = meshmod.decompose(8, 4, rank)
        lay = debug_layout(capi, mesh, True, 64)
        fs = _check_structure(mesh, lay)
        assert fs.nRecv > 0 and np.any(fs.li < fs.ls[1:])
        coef = meshmod.pressure_laplacian(mesh)
        recv = meshmod.cell_field_global(mesh, 21)[:fs.nRecv] * 0.5 - 0.125
        nr = [p.neighbRank for p in mesh.coupled_patches()]
        _check_replay(orc, meshmod, mesh, lay, coef, neighbRank=nr, comm_recv=recv)


def test_face_stream_cyclic(capi, orc, meshmod):
    from test_oracle_core import _cyclic_case
    m, c, ps, fc, nr, lo, hi = _cyclic_case(meshmod, "P")
    lay = debug_layout(capi, m, True, None, patches=(ps, fc))
    _check_structure(m, lay, patches=(ps, fc))
    _check_replay(orc, meshmod, m, lay, dict(diag=c["diag"], upper=c["upper"], bou=c["bou"]), patches=(ps, fc),
                  neighbRank=nr)


def test_face_stream_narrowed_bands(capi, orc):
    """A random graph without locality: the builder narrows the bands; the face stream stays exact."""
    from test_layout_cpu import _RandomGraph
    g = _RandomGraph(30000, 6, 1)
    lay = debug_layout(capi, g, centres=False, band=16384)
    assert int(lay["dims"][2]) < 16384
    _check_structure(g, lay)
    rng = np.random.default_rng(3)
    upper = rng.uniform(-1, 1, g.nFaces)
    diag = rng.uniform(2, 3, g.nCells)
    psi = rng.uniform(-1, 1, g.nCells)
    a = orc.Addr(g.nCells, g.lower, g.upper)
    ref = orc.Matrix(a, diag, upper, None).amul(psi)
    got = _replay_amul(lay, diag, upper, np.zeros(0), psi, np.zeros(0))
    assert np.array_equal(_bits(got), _bits(ref))


def test_face_stream_selection(capi, meshmod):
    """Large meshes use the face stream; its buffer never costs residency against the entry stream's tile."""
    mesh = meshmod.hex_mesh(64)
    lay = debug_layout(capi, mesh, True, 512)
    fs = _Fs(lay)
    assert fs.used == 1 and fs.nOwn >= mesh.nFaces
