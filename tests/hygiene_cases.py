"""Ragged and degenerate meshes for tests/test_gpu_memory_hygiene.py and tests/test_memory_hygiene_cpu.py: the sizes where the
banded layout's padding, the two-rows-per-lane staging, the persistent-CTA scheduling and the deterministic partial sums go wrong.
Every shape is a tests/polymesh_cases.PolyBox, so the builders of that module accept it.

    cell1          1 cell, no faces
    pair           2 cells, one face
    chainN         N cells in a row (N = 3, 63, 64, 65, 127, 129): the last 64-row slice one row long, an odd row in a lane's pair
    boxN           hex boxes of 64k +- 1 cells
    isolated       400 cells of which most have no face at all
    components     two disconnected hex boxes
    hub100/3000    one cell with 100 (3000) neighbours that form a chain among themselves
    cyclic2        2 cells with one face and a cyclic patch pair between them"""
import importlib

import numpy as np

import polymesh_cases as pc

meshmod = importlib.import_module("rapidcfd-dev_b200.mesh")

BOXES = {"box63": (7, 9, 1), "box65": (13, 5, 1), "box255": (17, 5, 3), "box513": (19, 9, 3), "box1023": (31, 11, 3)}
CHAINS = (3, 63, 64, 65, 127, 129)
NAMES = ["cell1", "pair"] + [f"chain{n}" for n in CHAINS] + list(BOXES) + ["isolated", "components", "hub100", "hub3000", "cyclic2"]
# the shapes with a finite-volume geometry worth the face sums, the fvMatrix glue and MULES
FV_NAMES = list(BOXES) + ["hub100", "hub3000"]


def _graph_box(nCells, lower, upper, seed, nB=None, patches=()):
    """PolyBox of an arbitrary LDU graph with random geometry (as polymesh_cases.graph) and an unsorted wall patch of nB faces"""
    lower, upper = np.asarray(lower, np.int32), np.asarray(upper, np.int32)
    assert np.all(lower < upper) and len(np.unique(lower.astype(np.int64) * nCells + upper)) == len(lower)
    o = np.lexsort((upper, lower))        # upper-triangular face order: owner ascending, then neighbour
    lower, upper = lower[o], upper[o]
    rng = np.random.default_rng(seed)
    nF = len(lower)
    nB = (nCells + 1) // 2 if nB is None else nB
    bfc = rng.integers(0, nCells, nB).astype(np.int32)
    walls = [pc.BPatch("walls", bfc, rng.uniform(-1, 1, (nB, 3)), rng.uniform(0, 1, (nB, 3)))]
    return pc.PolyBox(nCells, lower, upper, rng.uniform(0, 1, (nCells, 3)), rng.uniform(0.5, 2, nCells), rng.uniform(-1, 1, (nF, 3)),
                      rng.uniform(0, 1, (nF, 3)), rng.uniform(0.2, 0.8, nF), rng.uniform(1, 2, nF), walls + list(patches))


def _hex_box(dims, shift=0):
    """PolyBox of mesh.hex_mesh(*dims), cells numbered from `shift` (the geometry of a unit-spaced lattice)"""
    m = meshmod.hex_mesh(*dims)
    C = m.cell_centres()
    walls = []
    for p in m.wall_patches():
        n = p.Sf / np.sqrt((p.Sf ** 2).sum(1))[:, None]
        walls.append(pc.BPatch(p.name, p.faceCells.astype(np.int32) + shift, p.Sf, C[p.faceCells] + 0.5 * m.h * n))
    return m, C, walls


def _hex(dims):
    m, C, walls = _hex_box(dims)
    return pc.PolyBox(m.nCells, m.lower, m.upper, C, m.volumes(), m.Sf(), m.face_centres(), m.weights(), m.deltaCoeffs(), walls)


def _components():
    a, Ca, wa = _hex_box((4, 4, 4))
    b, Cb, wb = _hex_box((5, 3, 3), a.nCells)
    Cb = Cb + np.array([2.0, 0.0, 0.0])
    for p in wb:
        p.Cf = p.Cf + np.array([2.0, 0.0, 0.0])
    cat = np.concatenate
    return pc.PolyBox(a.nCells + b.nCells, cat([a.lower, b.lower + a.nCells]), cat([a.upper, b.upper + a.nCells]), cat([Ca, Cb]),
                      cat([a.volumes(), b.volumes()]), cat([a.Sf(), b.Sf()]), cat([a.face_centres(), b.face_centres() + [2.0, 0, 0]]),
                      cat([a.weights(), b.weights()]), cat([a.deltaCoeffs(), b.deltaCoeffs()]), wa + wb)


def _hub(k):
    """cell 0 owns a face to each of cells 1..k, which form a chain among themselves"""
    leaves = np.arange(1, k + 1)
    return _graph_box(k + 1, np.concatenate([np.zeros(k, np.int32), leaves[:-1]]), np.concatenate([leaves, leaves[1:]]), k)


def _isolated():
    rng = np.random.default_rng(17)
    cells = np.sort(rng.choice(400, 30, replace=False))
    pairs = {(int(min(a, b)), int(max(a, b))) for a, b in zip(cells[:-1], cells[1:])} | {(int(cells[0]), int(cells[-1]))}
    lo, up = zip(*sorted(pairs))
    return _graph_box(400, lo, up, 17)


def _cyclic2():
    rng = np.random.default_rng(5)
    cyc = [pc.BPatch("left", np.array([0], np.int32), np.array([[-1.0, 0, 0]]), np.array([[0.0, 0.5, 0.5]]), "cyclic", -2),
           pc.BPatch("right", np.array([1], np.int32), np.array([[1.0, 0, 0]]), np.array([[1.0, 0.5, 0.5]]), "cyclic", -1)]
    b = _graph_box(2, [0], [1], 5, nB=2, patches=cyc)
    b._C = np.array([[0.25, 0.5, 0.5], [0.75, 0.5, 0.5]])
    b._Sf = np.array([[1.0, 0.0, 0.0]]) + rng.uniform(-1e-3, 1e-3, (1, 3))
    return b


def build(name):
    if name == "cell1":
        return _graph_box(1, [], [], 1, nB=3)
    if name == "pair":
        return _graph_box(2, [0], [1], 2)
    if name.startswith("chain"):
        n = int(name[5:])
        return _graph_box(n, np.arange(n - 1), np.arange(1, n), n)
    if name in BOXES:
        return _hex(BOXES[name])
    return {"isolated": _isolated, "components": _components, "hub100": lambda: _hub(100), "hub3000": lambda: _hub(3000),
            "cyclic2": _cyclic2}[name]()


def coefficients(box, symmetric, seed=0):
    """(diag, upper, lower or None, bou, int) of a strictly diagonally dominant matrix on `box`: every solver converges on every
    component, isolated cells included; the coupled coefficients are None without a cyclic pair, one shared array when symmetric"""
    rng = np.random.default_rng(seed)
    nF = box.nFaces
    upper = -rng.uniform(0.5, 1.5, nF)
    lower = None if symmetric else upper * rng.uniform(0.3, 1.7, nF)
    off = np.zeros(box.nCells)
    np.add.at(off, box.lower, np.abs(upper))
    np.add.at(off, box.upper, np.abs(upper if lower is None else lower))
    ps, fc, nr, _ = box.coupled_arrays()
    bou = itc = None
    if fc is not None:
        bou = -rng.uniform(0.2, 0.6, len(fc))
        if symmetric:     # the faces of a cyclic pair carry one coefficient: face j of patch p is face j of its partner
            for p in range(len(nr)):
                q = -nr[p] - 1
                if q < p:
                    bou[ps[p]:ps[p + 1]] = bou[ps[q]:ps[q + 1]]
        itc = bou if symmetric else bou * rng.uniform(0.5, 1.5, len(fc))
        np.add.at(off, fc, np.abs(bou) + np.abs(itc))
    diag = off + box.volumes() * rng.uniform(0.5, 1.5, box.nCells)
    return diag, upper, lower, bou, itc


def oracle_matrix(orc, box, coeffs):
    diag, upper, lower, bou, itc = coeffs
    a = pc.addr(orc, box)
    return a, orc.Matrix(a, diag, upper, lower, bou, itc) if bou is not None else orc.Matrix(a, diag, upper, lower)
