"""OpenFOAM on-disk formats (rapidcfd-dev_b200/foamfile.py, SURVEY.md 8(f) rank 3): dictionary
syntax + look-up rules, fvSolution -> solver selection, polyMesh files (ascii / binary / gz,
processor and cyclic patches), geometry against analytic values and the divergence theorem, and an
unstructured-numbering case read from disk that drives the oracle and the banded-layout builder."""
import gzip
import importlib
import os
import shutil

import numpy as np
import pytest

from conftest import dense_from_ldu
from layout_helpers import debug_layout
from test_layout_cpu import _check_layout, capi  # noqa: F401  (capi is a fixture)


@pytest.fixture(scope="module")
def ff():
    return importlib.import_module("rapidcfd-dev_b200.foamfile")


FVSOLUTION = r'''
/*--------------------------------*- C++ -*----------------------------------*\
| a typical system/fvSolution                                                 |
\*---------------------------------------------------------------------------*/
FoamFile
{
    version     2.0;
    format      ascii;
    class       dictionary;
    location    "system";
    object      fvSolution;
}
// * * * * * * * * * * * * * * * * * * * * * * * * * * * * * * * * * * * * * //

tol 1e-06;

solvers
{
    p
    {
        solver          PCG;
        preconditioner  DIC;
        tolerance       $tol;
        relTol          0.05;   // trailing comment
    }

    pFinal
    {
        solver          GAMG;
        smoother        GaussSeidel;
        tolerance       1e-07;
        relTol          0;
        cacheAgglomeration on;
        agglomerator    faceAreaPair;
        nCellsInCoarsestLevel 20;
        mergeLevels     2;
        nPreSweeps      1;
        directSolveCoarsest no;
        scaleCorrection yes;
    }

    "(U|k|epsilon)"
    {
        solver          PBiCG;
        preconditioner  { preconditioner DILU; }
        tolerance       1e-05;
        relTol          0;
        maxIter         200;
    }

    "(U|k|epsilon)Final"
    {
        solver          smoothSolver;
        smoother        { smoother GaussSeidel; }
        nSweeps         2;
        tolerance       1e-08;
    }

    ".*"
    {
        solver          PBiCGStab;
        preconditioner  none;
    }

    T { solver ICCG; tolerance 1e-9; relTol 0; }
}

PISO
{
    nCorrectors     2;
    nNonOrthogonalCorrectors 0;
    pRefCell        0;
    pRefValue       0;
}

nu              nu [ 0 2 -1 0 0 0 0 ] 0.01;
vertices        ( (0 0 0) (1 0 0) (1 1 0) );
blocks          ( hex (0 1 2 3 4 5 6 7) (20 20 1) simpleGrading (1 1 1) );
'''


def test_dictionary_syntax_and_lookup(ff):
    d = ff.parse_dict(FVSOLUTION, "fvSolution")
    assert d.toc()[:2] == ["FoamFile", "tol"]
    assert d.subDict("FoamFile").lookup("class") == "dictionary"
    piso = d.subDict("PISO")
    assert piso.lookup("nCorrectors") == 2 and piso.lookupOrDefault("momentumPredictor", "on") == "on"
    assert d.lookup("nu") == ["nu", [0, 2, -1, 0, 0, 0, 0], 0.01]
    assert d.lookup("vertices") == [[0, 0, 0], [1, 0, 0], [1, 1, 0]]
    assert d.lookup("blocks")[0] == "hex" and d.lookup("blocks")[2] == [20, 20, 1]
    s = d.subDict("solvers")
    assert s.subDict("p").lookup("tolerance") == 1e-06          # $tol expanded from the enclosing scope
    # exact keyword wins over patterns; among patterns the most recently defined one wins (dictionary.C:313-316)
    assert s.subDict("U").lookup("solver") == "PBiCGStab"       # ".*" was defined after "(U|k|epsilon)"
    assert s.subDict("p").lookup("solver") == "PCG"
    with pytest.raises(KeyError, match="undefined"):
        piso.lookup("nOuterCorrectors")
    with pytest.raises(KeyError, match="not a sub-dictionary"):
        d.subDict("tol")
    with pytest.raises(ValueError):
        ff.parse_dict("a { b 1; ")
    with pytest.raises(ValueError):
        ff.parse_dict("a 1")
    with pytest.raises(ValueError, match="not supported"):
        ff.parse_dict('#include "other";')


def test_fvsolution_solver_selection(ff):
    text = FVSOLUTION.replace('    ".*"\n    {\n        solver          PBiCGStab;\n        preconditioner  none;\n    }\n', "")
    d = ff.parse_dict(text)
    assert ff.solver_controls(d, "p") == ("PCG", "DIC", dict(tolerance=1e-06, relTol=0.05))
    sv, sm, c = ff.solver_controls(d, "pFinal")
    assert (sv, sm) == ("GAMG", "GaussSeidel")
    assert c == dict(tolerance=1e-07, relTol=0.0, nCellsInCoarsestLevel=20, mergeLevels=2, nPreSweeps=1,
                     directSolveCoarsest=0, scaleCorrection=1)
    for fld in ("U", "k", "epsilon"):
        assert ff.solver_controls(d, fld) == ("PBiCG", "DILU", dict(tolerance=1e-05, relTol=0.0, maxIter=200))
    assert ff.solver_controls(d, "UFinal") == ("smoothSolver", "GaussSeidel", dict(tolerance=1e-08, nSweeps=2))
    assert ff.solver_controls(d, "T") == ("ICCG", "DIC", dict(tolerance=1e-9, relTol=0.0))
    with pytest.raises(KeyError):
        ff.solver_controls(d, "omega")


def test_controls_feed_the_oracle(ff, meshmod, orc):
    """the parsed controls select and drive a solve exactly like hand-written keyword arguments"""
    d = ff.parse_dict(FVSOLUTION)
    m = meshmod.hex_mesh(8, 8, 8)
    c = meshmod.pressure_laplacian(m)
    M = orc.Matrix(orc.Addr(m.nCells, m.lower, m.upper), c["diag"], c["upper"], None)
    b = M.amul(meshmod.cell_field_global(m, 42))
    sv, pre, ctl = ff.solver_controls(d, "p")
    psi1, p1, h1 = M.solve(sv, pre, np.zeros(m.nCells), b, **ctl)
    psi2, p2, h2 = M.solve("PCG", "DIC", np.zeros(m.nCells), b, tolerance=1e-6, relTol=0.05)
    assert p1.nIterations == p2.nIterations and np.array_equal(psi1, psi2)
    assert p1.solverName == b"AINVPCG"


@pytest.mark.parametrize("binary", [False, True])
def test_polymesh_roundtrip_and_geometry(ff, meshmod, tmp_path, binary):
    hm = meshmod.hex_mesh(5, 4, 3)
    pm = ff.from_hex_mesh(hm)
    d = str(tmp_path / "constant" / "polyMesh")
    ff.write_poly_mesh(d, pm, binary)
    # neighbour compressed: the reader falls back to <name>.gz like OpenFOAM does
    with open(os.path.join(d, "neighbour"), "rb") as f, gzip.open(os.path.join(d, "neighbour.gz"), "wb") as g:
        shutil.copyfileobj(f, g)
    os.remove(os.path.join(d, "neighbour"))
    r = ff.read_poly_mesh(d)
    lo, up = r.ldu()
    assert np.array_equal(lo, hm.lower) and np.array_equal(up, hm.upper) and r.nCells == hm.nCells
    assert [(p.name, p.type, p.nFaces) for p in r.patches] == [(p.name, "wall", len(p.faceCells)) for p in hm.patches]
    assert r.coupled_interface_arrays() == (None, None, None)
    assert np.array_equal(r.boundary_face_cells(), np.concatenate([p.faceCells for p in hm.patches]))
    g = r.fv_geometry()
    np.testing.assert_allclose(g["C"], hm.cell_centres(), atol=1e-15)
    np.testing.assert_allclose(g["V"], hm.volumes(), rtol=1e-14)
    np.testing.assert_allclose(g["Sf"][:hm.nFaces], hm.Sf(), atol=1e-16)
    np.testing.assert_allclose(g["weights"], 0.5, rtol=1e-14)
    np.testing.assert_allclose(g["deltaCoeffs"], 1.0 / hm.h, rtol=1e-14)
    for p, q in zip(hm.patches, r.patches):
        np.testing.assert_allclose(g["Sf"][q.startFace:q.startFace + q.nFaces], p.Sf, atol=1e-16)


def test_decomposed_case_processor_patches(ff, meshmod, tmp_path):
    """processorN/constant/polyMesh of a 2x2x1 decomposition: the coupled-patch arrays handed to
    b200ldu_addr_create equal those of the in-memory decomposition."""
    for rank in range(4):
        hm = meshmod.decompose(8, 4, rank)
        d = str(tmp_path / f"processor{rank}" / "constant" / "polyMesh")
        ff.write_poly_mesh(d, ff.from_hex_mesh(hm, rank))
        r = ff.read_poly_mesh(d, geometry=False)
        ps, fc, nr = r.coupled_interface_arrays()
        eps, efc = hm.patch_start_facecells()
        assert np.array_equal(ps, eps) and np.array_equal(fc, efc)
        assert nr.tolist() == [p.neighbRank for p in hm.coupled_patches()]
        assert all(p.myProcNo == rank for p in r.patches if p.type == "processor")
        assert r.points is None


def test_cyclic_patches_from_boundary_file(ff, meshmod, tmp_path):
    hm = meshmod.hex_mesh(6, 5, 4)
    pm = ff.from_hex_mesh(hm)
    names = [p.name for p in pm.patches]
    a, b = pm.patches[0], pm.patches[1]          # x-min / x-max walls become a cyclic pair
    a.type = b.type = "cyclic"
    a.neighbourPatch, b.neighbourPatch = b.name, a.name
    d = str(tmp_path / "polyMesh")
    ff.write_poly_mesh(d, pm)
    r = ff.read_poly_mesh(d)
    ps, fc, nr = r.coupled_interface_arrays()
    assert nr.tolist() == [-2, -1] and ps.tolist() == [0, 20, 40]
    assert np.array_equal(fc[:20], hm.patches[0].faceCells) and np.array_equal(fc[20:], hm.patches[1].faceCells)
    assert [p.name for p in r.patches] == names
    b.neighbourPatch = "nowhere"
    ff.write_poly_mesh(d, pm)
    with pytest.raises(ValueError, match="neighbourPatch"):
        ff.read_poly_mesh(d).coupled_interface_arrays()


def _scrambled(ff, meshmod, dims, seed, skew=0.25):
    """hex cells renumbered at random (faces re-sorted into upper-triangular order) with skewed
    points: an unstructured-numbering, non-orthogonal mesh as a mesher would write it."""
    hm = meshmod.hex_mesh(*dims)
    pm = ff.from_hex_mesh(hm)
    rng = np.random.default_rng(seed)
    new = rng.permutation(hm.nCells).astype(np.int32)       # old cell -> new cell
    nI = pm.nInternalFaces
    own, nei = new[pm.owner[:nI]], new[pm.neighbour]
    flip = own > nei
    o2, n2 = np.where(flip, nei, own), np.where(flip, own, nei)
    order = np.lexsort((n2, o2))
    quads = pm.faceLabels.reshape(-1, 4).copy()
    qi = quads[:nI]
    qi[flip] = qi[flip][:, ::-1]                               # keep the normal pointing owner -> neighbour
    quads[:nI] = qi[order]
    owner = np.concatenate([o2[order], new[pm.owner[nI:]]]).astype(np.int32)
    pts = pm.points.copy()
    interior = np.all((pts > 1e-12) & (pts < np.array([1.0, dims[1] / dims[0], dims[2] / dims[0]]) - 1e-12), axis=1)
    pts[interior] += skew * hm.h * (rng.random((int(interior.sum()), 3)) - 0.5)
    return ff.PolyMesh(owner, n2[order].astype(np.int32), pm.patches, pts, pm.faceOffsets,
                       quads.reshape(-1).astype(np.int32)), hm


def test_geometry_divergence_theorem_on_skewed_mesh(ff, meshmod):
    pm, hm = _scrambled(ff, meshmod, (6, 5, 4), 3)
    g = pm.fv_geometry()
    nI = pm.nInternalFaces
    closed = np.zeros((pm.nCells, 3))                          # sum of outward area vectors of every cell
    np.add.at(closed, pm.owner, g["Sf"])
    np.subtract.at(closed, pm.neighbour, g["Sf"][:nI])
    np.testing.assert_allclose(closed, 0, atol=1e-15)
    np.testing.assert_allclose(g["V"].sum(), hm.nCells * hm.h ** 3, rtol=1e-13)
    vol = np.zeros(pm.nCells)                                  # V = 1/3 sum Cf.Sf (Gauss)
    np.add.at(vol, pm.owner, np.einsum("ij,ij->i", g["Cf"], g["Sf"]) / 3)
    np.subtract.at(vol, pm.neighbour, np.einsum("ij,ij->i", g["Cf"][:nI], g["Sf"][:nI]) / 3)
    np.testing.assert_allclose(g["V"], vol, rtol=1e-12)
    assert np.all(g["V"] > 0) and np.all((g["weights"] > 0.2) & (g["weights"] < 0.8))
    d = g["C"][pm.neighbour] - g["C"][pm.owner[:nI]]
    assert np.all(np.einsum("ij,ij->i", d, g["Sf"][:nI]) > 0)  # normals point owner -> neighbour


class _AsMesh:
    """adapter: PolyMesh -> what tests/test_layout_cpu.py expects of a mesh"""

    def __init__(self, pm, centres):
        self.lower, self.upper = pm.ldu()
        self.nCells, self.nFaces = pm.nCells, len(self.lower)
        self._c = centres
        self._pm = pm

    def cell_centres(self):
        return self._c

    def patch_start_facecells(self):
        ps, fc, _ = self._pm.coupled_interface_arrays()
        if ps is None:
            return np.zeros(1, np.int32), np.zeros(0, np.int32)
        return ps, fc


@pytest.mark.parametrize("centres", [True, False])
def test_unstructured_case_from_disk_drives_oracle_and_layout(ff, meshmod, orc, capi, tmp_path, centres):  # noqa: F811
    """A randomly numbered, skewed mesh written to constant/polyMesh, read back, assembled into the
    Laplacian from its own geometry (gaussLaplacianScheme: upper = deltaCoeffs*|Sf|), solved by the
    oracle against a dense solve, and banded by the product's layout builder (with cell centres and
    with the graph-distance embedding) -- structural check face for face."""
    pm0, hm = _scrambled(ff, meshmod, (7, 6, 5), 11)
    d = str(tmp_path / "constant" / "polyMesh")
    ff.write_poly_mesh(d, pm0, binary=True)
    pm = ff.read_poly_mesh(d)
    g = pm.fv_geometry()
    lo, up = pm.ldu()
    upper = g["deltaCoeffs"] * g["magSf"][:len(lo)]
    diag = np.zeros(pm.nCells)
    np.subtract.at(diag, lo, upper)
    np.subtract.at(diag, up, upper)
    diag[0] *= 2
    a = orc.Addr(pm.nCells, lo, up)
    M = orc.Matrix(a, diag, upper, None)
    A = dense_from_ldu(pm.nCells, lo, up, diag, upper)
    xs = np.random.default_rng(2).standard_normal(pm.nCells)
    b = A @ xs
    np.testing.assert_allclose(M.amul(xs), b, rtol=1e-12, atol=1e-12)
    psi, perf, _ = M.solve("PCG", "DIC", np.zeros(pm.nCells), b, tolerance=1e-10, maxIter=500)
    assert perf.converged
    np.testing.assert_allclose(psi, xs, atol=1e-6)
    mesh = _AsMesh(pm, g["C"] if centres else None)
    lay = debug_layout(capi, mesh, centres=centres, band=64)
    _check_layout(mesh, lay)
    nPad, nBands, bandRows, nRecv, maxHalo = [int(x) for x in lay["dims"]]
    assert nBands >= 3 and maxHalo < 4 * bandRows      # the renumbering keeps the bands compact


def test_decompose_poly_mesh_matches_brick_decomposition(ff, meshmod, orc, tmp_path):
    """decomposePar-style splitting of a polyMesh by a cell -> rank map: for the 2x2x1 brick map it gives
    the in-memory decomposition of mesh.decompose (same local addressing, processor patches in the same
    order with the same face order on both sides); geometry of the pieces is consistent (flipped faces
    point out of their new owner); a decomposed PCG solve through files equals the single-domain one."""
    import dist_helpers as dh
    n, nR = 8, 4
    g = meshmod.hex_mesh(n)
    pm = ff.from_hex_mesh(g)
    px, py, pz = meshmod.brick_split(nR)
    c = np.arange(g.nCells)
    i, j, k = c % n, (c // n) % n, c // (n * n)
    proc = (i // (n // px)) + px * (j // (n // py)) + px * py * (k // (n // pz))
    parts = ff.decompose_poly_mesh(pm, proc)
    assert len(parts) == nR
    for r, (sub, cells, faceG) in enumerate(parts):
        hm = meshmod.decompose(n, nR, r)
        assert np.array_equal(cells, hm.cellGlobal)
        lo, up = sub.ldu()
        assert np.array_equal(lo, hm.lower) and np.array_equal(up, hm.upper)
        ps, fc, nr = sub.coupled_interface_arrays()
        eps, efc = hm.patch_start_facecells()
        assert np.array_equal(ps, eps) and np.array_equal(fc, efc)
        assert nr.tolist() == [p.neighbRank for p in hm.coupled_patches()]
        d = str(tmp_path / f"processor{r}" / "constant" / "polyMesh")
        ff.write_poly_mesh(d, sub, binary=(r % 2 == 0))
        back = ff.read_poly_mesh(d)
        geo = back.fv_geometry()
        np.testing.assert_allclose(geo["C"], hm.cell_centres(), atol=1e-14)
        np.testing.assert_allclose(geo["V"], hm.volumes(), rtol=1e-13)
        for p in back.patches:                     # every boundary face points out of its (new) owner
            f = np.arange(p.startFace, p.startFace + p.nFaces)
            out = geo["Cf"][f] - geo["C"][back.owner[f]]
            assert np.all(np.einsum("ij,ij->i", out, geo["Sf"][f]) > 0)
    # the two sides of every processor patch list the same global faces in the same order
    for r, (sub, cells, faceG) in enumerate(parts):
        for p in sub.patches:
            if p.type != "processor":
                continue
            mine = faceG[p.startFace:p.startFace + p.nFaces]
            osub, _, oG = parts[p.neighbProcNo]
            q = [x for x in osub.patches if x.type == "processor" and x.neighbProcNo == r][0]
            theirs = oG[q.startFace:q.startFace + q.nFaces]
            gm = np.where(mine >= 0, mine, -mine - 1)
            gt = np.where(theirs >= 0, theirs, -theirs - 1)
            assert np.array_equal(gm, gt) and np.all((mine >= 0) != (theirs >= 0))
    # solve through the decomposed files (threads as ranks) == single domain, with the diagonal preconditioner
    gm_, gc_ = dh.global_case(meshmod, n, "P")
    ga, gM = dh.oracle_matrix(orc, gm_, gc_)
    xs = meshmod.cell_field_global(gm_, 42)
    b = gM.amul(xs)
    psi_ref, pref, href = gM.solve("PCG", "diagonal", np.zeros(g.nCells), b, tolerance=1e-9, maxIter=500)
    ex = dh.ThreadExchange(nR)

    def rank_fn(r):
        hm, coef = dh.local_case(meshmod, n, nR, r, "P")           # coefficients of the local piece
        sub = ff.read_poly_mesh(str(tmp_path / f"processor{r}" / "constant" / "polyMesh"), geometry=False)
        lo, up = sub.ldu()
        ps, fc, nr = sub.coupled_interface_arrays()
        a = orc.Addr(sub.nCells, lo, up, ps, fc, neighbRank=nr)    # addressing straight from the files
        M = orc.Matrix(a, coef["diag"], coef["upper"], coef["lower"], coef["bou"], coef["int"])
        comm = ex.comm(orc, r, hm, n ** 3)
        psi, perf, hist = M.solve("PCG", "diagonal", np.zeros(sub.nCells), b[hm.cellGlobal], comm=comm,
                                  tolerance=1e-9, maxIter=500)
        return hm.cellGlobal, psi, perf.nIterations, hist
    res = dh.run_threads(nR, rank_fn)
    for cg, psi, nit, hist in res:
        assert abs(nit - pref.nIterations) <= 1
        np.testing.assert_allclose(psi, psi_ref[cg], atol=1e-7)
        np.testing.assert_allclose(hist[:25], href[:25], rtol=1e-9)


# ---- property tests (hypothesis): list files and dictionaries survive a write/parse round trip ----
from hypothesis import given, settings, strategies as st  # noqa: E402


@settings(max_examples=40, deadline=None)
@given(st.lists(st.integers(min_value=-2**31, max_value=2**31 - 1), max_size=60), st.booleans())
def test_label_list_roundtrip(tmp_path_factory, values, binary):
    ff = importlib.import_module("rapidcfd-dev_b200.foamfile")
    p = str(tmp_path_factory.mktemp("ll") / "owner")
    ff.write_list(p, "label", np.array(values, dtype=np.int64), binary)
    assert ff.read_list(p, "label").tolist() == values


@settings(max_examples=40, deadline=None)
@given(st.lists(st.tuples(*[st.floats(allow_nan=False, allow_infinity=False, width=64)] * 3), max_size=40), st.booleans())
def test_vector_list_roundtrip_is_exact(tmp_path_factory, values, binary):
    ff = importlib.import_module("rapidcfd-dev_b200.foamfile")
    p = str(tmp_path_factory.mktemp("vl") / "points")
    a = np.array(values, dtype=np.float64).reshape(-1, 3)
    ff.write_list(p, "vector", a, binary)
    back = ff.read_list(p, "vector")
    assert back.shape == a.shape and np.array_equal(back, a)      # repr() round-trips doubles exactly


@settings(max_examples=40, deadline=None)
@given(st.lists(st.lists(st.integers(min_value=0, max_value=10**6), min_size=3, max_size=9), max_size=30), st.booleans())
def test_face_list_roundtrip(tmp_path_factory, faces, binary):
    ff = importlib.import_module("rapidcfd-dev_b200.foamfile")
    p = str(tmp_path_factory.mktemp("fl") / "faces")
    offs = np.concatenate([[0], np.cumsum([len(f) for f in faces])]).astype(np.int32)
    labels = np.array([v for f in faces for v in f], dtype=np.int32)
    ff.write_list(p, "face", (offs, labels), binary)
    o2, l2 = ff.read_list(p, "face")
    assert np.array_equal(o2, offs) and np.array_equal(l2, labels)


_word = st.text(alphabet="abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ_", min_size=1, max_size=8)
_scalar = st.one_of(st.integers(min_value=-10**6, max_value=10**6),
                    st.floats(allow_nan=False, allow_infinity=False, min_value=-1e12, max_value=1e12), _word)
# lists are homogeneous (all scalars or all lists): `N ( ... )` is OpenFOAM's sized-list notation, so an integer
# directly followed by a list inside a list is genuinely ambiguous and not generated
_value = st.one_of(_scalar, st.lists(_scalar, max_size=4), st.lists(st.lists(_scalar, max_size=3), max_size=3))
_dict = st.recursive(st.dictionaries(_word, _value, max_size=4),
                     lambda inner: st.dictionaries(_word, st.one_of(_value, inner), max_size=4), max_leaves=10)


def _emit(d, ind=0):
    pad = "    " * ind
    out = []
    for k, v in d.items():
        if isinstance(v, dict):
            out.append(f"{pad}{k}\n{pad}{{\n{_emit(v, ind + 1)}{pad}}}\n")
        else:
            out.append(f"{pad}{k} {_emit_value(v)};   // c\n")
    return "".join(out)


def _emit_value(v):
    if isinstance(v, list):
        return "( " + " ".join(_emit_value(x) for x in v) + " )"
    return repr(v) if isinstance(v, float) else str(v)


@settings(max_examples=60, deadline=None)
@given(_dict)
def test_dictionary_roundtrip(d):
    ff = importlib.import_module("rapidcfd-dev_b200.foamfile")
    text = "/* header */\n" + _emit(d)
    assert ff.parse_dict(text).to_python() == d


@pytest.mark.parametrize("binary", [False, True])
def test_field_files_roundtrip(ff, tmp_path, binary):
    """0/p and 0/U as icoFoam's cavity case has them (uniform internal fields, fixedValue lid) and a
    restart-style nonuniform pair, ascii and binary."""
    rng = np.random.default_rng(0)
    n = 12
    p_bf = {"movingWall": {"type": "zeroGradient"}, "fixedWalls": {"type": "zeroGradient"}, "frontAndBack": {"type": "empty"}}
    U_bf = {"movingWall": {"type": "fixedValue", "value": np.array([1.0, 0.0, 0.0])},
            "fixedWalls": {"type": "fixedValue", "value": np.array([0.0, 0.0, 0.0])}, "frontAndBack": {"type": "empty"}}
    ff.write_field(str(tmp_path / "p"), "volScalarField", [0, 2, -2, 0, 0, 0, 0], 0.0, p_bf, binary)
    ff.write_field(str(tmp_path / "U"), "volVectorField", [0, 1, -1, 0, 0, 0, 0], np.zeros(3), U_bf, binary)
    p = ff.read_field(str(tmp_path / "p"), nInternal=n)
    U = ff.read_field(str(tmp_path / "U"), nInternal=n)
    assert p["cls"] == "volScalarField" and p["dimensions"] == [0, 2, -2, 0, 0, 0, 0]
    assert p["internalField"].shape == (n,) and not p["internalField"].any()
    assert U["internalField"].shape == (n, 3) and U["boundaryField"]["movingWall"]["type"] == "fixedValue"
    assert np.array_equal(U["boundaryField"]["movingWall"]["value"], [1.0, 0.0, 0.0])
    assert p["boundaryField"]["frontAndBack"] == {"type": "empty"}
    pv, Uv = rng.standard_normal(n), rng.standard_normal((n, 3))
    lid = rng.standard_normal((4, 3))
    U_bf["movingWall"]["value"] = lid
    ff.write_field(str(tmp_path / "p1"), "volScalarField", [0, 2, -2, 0, 0, 0, 0], pv, p_bf, binary)
    ff.write_field(str(tmp_path / "U1"), "volVectorField", [0, 1, -1, 0, 0, 0, 0], Uv, U_bf, binary)
    p1, U1 = ff.read_field(str(tmp_path / "p1")), ff.read_field(str(tmp_path / "U1"))
    assert np.array_equal(p1["internalField"], pv) and np.array_equal(U1["internalField"], Uv)
    assert np.array_equal(U1["boundaryField"]["movingWall"]["value"], lid)
    assert np.array_equal(U1["boundaryField"]["fixedWalls"]["value"], [0.0, 0.0, 0.0])


def test_fvSchemes_lookups_follow_the_reference():
    """fvSchemes.C:36-256, :425-580: per-kind default, `default none`, regular-expression keywords, the sections that default when
    missing, fluxRequired; keywords with balanced parentheses are single words (ISstream::read(word&))"""
    ff = importlib.import_module("rapidcfd-dev_b200.foamfile")
    d = ff.parse_dict("""
ddtSchemes { default Euler; }
gradSchemes { default Gauss linear; grad(p) leastSquares; }
divSchemes { default none; div(phi,U) Gauss limitedLinearV 1; div((nuEff*dev(T(grad(U))))) Gauss linear;
             "div\\(phi,(k|epsilon)\\)" bounded Gauss upwind; div(phi,alpha) Gauss vanLeer; }
laplacianSchemes { default Gauss linear corrected; }
fluxRequired { default no; p; }
""")
    assert ff.tokenize("div((nuEff*dev(T(grad(U))))) Gauss linear; f (1 2 3); g 2(4 5);") == [
        "div((nuEff*dev(T(grad(U)))))", "Gauss", "linear", ";", "f", "(", "1", "2", "3", ")", ";", "g", "2", "(", "4", "5", ")", ";"]
    s = ff.FvSchemes(d)
    assert s.ddt("ddt(U)") == ["Euler"] and s.grad("grad(U)") == ["Gauss", "linear"] and s.grad("grad(p)") == ["leastSquares"]
    assert s.div("div(phi,U)") == ["Gauss", "limitedLinearV", 1] and s.div("div((nuEff*dev(T(grad(U)))))") == ["Gauss", "linear"]
    assert s.div("div(phi,epsilon)") == ["bounded", "Gauss", "upwind"]
    assert s.laplacian("laplacian(nu,U)") == ["Gauss", "linear", "corrected"]
    assert s.interpolation("interpolate(U)") == ["linear"] and s.snGrad("snGrad(p)") == ["corrected"]     # missing sections
    assert s.fluxRequired("p") and not s.fluxRequired("U")
    with pytest.raises(KeyError, match="keyword div\\(phi,T\\) is undefined"):
        s.div("div(phi,T)")
    assert ff.convection_scheme(s.div("div(phi,k)")) == ("upwind", 1.0, True)
    assert ff.convection_scheme(["Gauss", "limitedLinear", 0.33]) == ("limitedLinear", 0.33, False)
    with pytest.raises(ValueError, match="Unknown discretisation scheme QUICK"):
        ff.convection_scheme(["Gauss", "QUICK"])
    with pytest.raises(ValueError, match="Unknown convection type"):
        ff.convection_scheme(["linear"])
