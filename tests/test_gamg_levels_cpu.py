"""GAMG level by level without a GPU.

 * The numpy restatement of the coarsest-level inverse (tests/gamg_levels.gj_inverse) equals the library's own host
   Gauss-Jordan (b200ldu_gamg_debug_invert, the code a device solve runs before it uploads the inverse) bit for bit, row
   swaps included, and meets the backward-error bound on the coarsest matrix of every case.
 * The oracle's opt-in device-coarsest mode, given that inverse, converges like its LU.
 * The coarse addressing of the host-only hierarchy read back through b200ldu_gamg_debug_get -- owner, neighbour, face
   restrict map and flips -- equals the oracle's on every level.
 * The oracle's coarse-matrix accessor equals the plain summation the reference's own functors are pinned to
   (oracle/ref_ldu.coarse_matrix)."""
import ctypes as C
import importlib
import types

import numpy as np
import pytest

import gamg_levels as gl
from layout_helpers import debug_addr, debug_lib
from oracle import ref_ldu

CASES = [("P", (16, 14, 12), 1), ("P", (16, 14, 12), 2), ("P", (16, 14, 12), 3), ("U", (16, 14, 12), 1),
         ("U", (16, 14, 12), 2), ("U", (16, 14, 12), 3), ("P", (9, 9, 9), 1), ("U", (9, 9, 9), 1),
         ("P", (9, 9, 9), 2), ("U", (9, 9, 9), 3), ("Uconv", (9, 9, 9), 1), ("Uconv", (16, 14, 12), 2)]


@pytest.fixture(scope="module")
def capi():
    g = importlib.import_module("__graft_entry__")
    g.build()
    return importlib.import_module("rapidcfd-dev_b200.capi")


def coefficients(meshmod, m, kind):
    if kind == "P":
        return meshmod.pressure_laplacian(m)
    if kind == "Uconv":  # convection-dominated: off-diagonals far above the diagonal, so the elimination pivots
        return meshmod.momentum_matrix(m, nu=1e-6, Co=50.0)
    return meshmod.momentum_matrix(m)


def oracle_case(meshmod, orc, kind, dims, merge):
    m = meshmod.hex_mesh(*dims)
    c = coefficients(meshmod, m, kind)
    oa = orc.Addr(m.nCells, m.lower, m.upper)
    om = orc.Matrix(oa, c["diag"], c["upper"], c["lower"])
    og = orc.Gamg(oa, meshmod.face_area_pair_weights(m), 10, mergeLevels=merge)
    return m, c, om, og


def coarsest_dense(og, om, perm=None):
    lev = og.nLevels - 1
    cm = og.coarse_matrix(om, lev)
    la = og.level_addr(lev)
    n = og.ncells(lev)
    return gl.banded_matrix(la.lower(), la.upper(), cm["diag"], cm["upper"], cm["lower"],
                            np.arange(n) if perm is None else perm)


def library_inverse(capi, A):
    N = A.shape[0]
    A = np.ascontiguousarray(A, np.float64)
    out = np.zeros((N, N))
    rc = capi.lib().b200ldu_gamg_debug_invert(N, A.ctypes.data, out.ctypes.data)
    return out, rc


@pytest.mark.parametrize("kind,dims,merge", CASES)
def test_gj_inverse_is_the_library_inverse_and_backward_stable(capi, meshmod, orc, kind, dims, merge):
    m, c, om, og = oracle_case(meshmod, orc, kind, dims, merge)
    n = og.ncells(og.nLevels - 1)
    rng = np.random.default_rng(7)
    for perm in (np.arange(n), rng.permutation(n)):
        A = coarsest_dense(og, om, perm)
        inv, swaps = gl.gj_inverse(A)
        lib_inv, lib_swaps = library_inverse(capi, A)
        assert lib_swaps == swaps
        assert gl.first_difference(inv, lib_inv) is None, gl.first_difference(inv, lib_inv)
        for b in (rng.standard_normal(n), np.abs(rng.standard_normal(n)), A @ np.ones(n)):
            x = gl.inverse_apply(inv, b)
            assert gl.backward_error(A, x, b) <= gl.BACKWARD_ERROR_BOUND
    if kind == "Uconv":
        assert swaps > 0  # the case exists to exercise the row swaps


@pytest.mark.parametrize("A", [
    [[1.0, 2.0, 0.0], [2.0, 1.0, 3.0], [-2.0, 0.0, 1.0]],         # tie in column 0 below the diagonal
    [[-3.0, 1.0, 1.0], [3.0, 2.0, 0.0], [0.0, 3.0, 5.0]],         # tie with the diagonal itself: no swap
    [[0.0, 1.0, 2.0], [4.0, 0.0, 1.0], [-4.0, 1.0, 0.0]],         # zero diagonal, tied candidates
    [[1e-300, 1.0], [1.0, 1e-300]]])
def test_gj_inverse_pivot_ties(capi, A):
    """The pivot search keeps the first of equal magnitudes; a restatement with >= (or any other tie rule) differs."""
    A = np.array(A)
    inv, swaps = gl.gj_inverse(A)
    lib_inv, lib_swaps = library_inverse(capi, A)
    assert lib_swaps == swaps
    assert gl.first_difference(inv, lib_inv) is None, gl.first_difference(inv, lib_inv)


def test_library_inverse_refuses_singular(capi):
    A = np.array([[1.0, 2.0], [2.0, 4.0]])
    assert library_inverse(capi, A)[1] == -1  # B200LDU_EINVAL


@pytest.mark.parametrize("kind,dims,merge", [c for c in CASES if c[0] != "Uconv"])  # GAMG does not converge there
def test_oracle_device_coarsest_mode_converges_like_lu(meshmod, orc, kind, dims, merge):
    m, c, om, og = oracle_case(meshmod, orc, kind, dims, merge)
    b = om.amul(meshmod.cell_field_global(m, 42))
    ctl = dict(tolerance=1e-9, maxIter=200, scaleCorrection=0)
    psi_lu, p_lu, h_lu = og.solve(om, "GaussSeidel", np.zeros(m.nCells), b, **ctl)
    n = og.ncells(og.nLevels - 1)
    perm = np.random.default_rng(3).permutation(n).astype(np.int32)
    inv, _ = gl.gj_inverse(coarsest_dense(og, om, perm))
    og.set_coarsest_inverse(inv, perm)
    psi_gj, p_gj, h_gj = og.solve(om, "GaussSeidel", np.zeros(m.nCells), b, **ctl)
    assert p_gj.converged and p_lu.converged
    assert p_gj.nIterations == p_lu.nIterations
    np.testing.assert_allclose(h_gj, h_lu, rtol=1e-6)
    np.testing.assert_allclose(psi_gj, psi_lu, rtol=0, atol=1e-10)
    # the mode applies what it was given: a wrong inverse changes the cycle (little, where many levels of smoothing
    # follow the coarsest solve of a diagonally dominant matrix)
    og.set_coarsest_inverse(inv * 2, perm)
    psi_bad, _, _ = og.solve(om, "GaussSeidel", np.zeros(m.nCells), b, **dict(ctl, maxIter=1))
    og.set_coarsest_inverse(inv, perm)
    psi_one, _, _ = og.solve(om, "GaussSeidel", np.zeros(m.nCells), b, **dict(ctl, maxIter=1))
    assert not np.array_equal(psi_bad, psi_one)
    # and None restores the LU, bit for bit
    og.set_coarsest_inverse(None)
    psi_lu2, _, _ = og.solve(om, "GaussSeidel", np.zeros(m.nCells), b, **ctl)
    assert np.array_equal(psi_lu2, psi_lu)


def _host_gamg(capi, m, w, merge, forward=1):
    h = debug_addr(capi, m, True)
    gg = capi.GamgAgglomeration(types.SimpleNamespace(h=h, nCells=m.nCells), w, 10, mergeLevels=merge, forward=forward)
    return h, gg


@pytest.mark.parametrize("dims,merge", [((16, 14, 12), 1), ((16, 14, 12), 2), ((16, 14, 12), 3), ((9, 9, 9), 1),
                                        ((9, 9, 9), 2), ((9, 9, 9), 3), ((7, 5, 3), 1)])
def test_host_coarse_addressing_is_the_oracles(capi, meshmod, orc, dims, merge):
    m = meshmod.hex_mesh(*dims)
    w = meshmod.face_area_pair_weights(m)
    og = orc.Gamg(orc.Addr(m.nCells, m.lower, m.upper), w, 10, mergeLevels=merge)
    h, gg = _host_gamg(capi, m, w, merge)
    try:
        assert gg.nLevels == og.nLevels > 0
        flipped = 0
        for lev in range(gg.nLevels):
            got, la = gg.level_addressing(lev), og.level_addr(lev)
            for name, ref in (("owner", la.lower()), ("neighbour", la.upper()),
                              ("faceRestrict", og.face_restrict_addr(lev)), ("faceFlip", og.face_flip(lev))):
                d = gl.first_difference(got[name], np.asarray(ref, np.int32), exact_int=True)
                assert d is None, f"level {lev} {name}: {d}"
            flipped += int(got["faceFlip"].sum())
        if dims == (9, 9, 9):
            assert flipped > 0  # the flip map is exercised, not all zeros
        # what a host-only hierarchy does not have
        for name in ("diag", "perm", "inv"):
            with pytest.raises(capi.B200LduError):
                gg.debug_get(gg.nLevels - 1, name)
        with pytest.raises(capi.B200LduError):
            gg.debug_get(gg.nLevels, "owner")
        L = capi.lib()
        assert L.b200ldu_gamg_debug_get(gg.h, 0, 12, None, 0) == -1
        assert L.b200ldu_gamg_debug_get(gg.h, -1, 0, None, 0) == -1
        # a short buffer gets the first cap elements and the full count back
        full = gg.debug_get(0, "faceRestrict")
        part = np.full(3, 7, np.int32)
        assert L.b200ldu_gamg_debug_get(gg.h, 0, 2, part.ctypes.data_as(C.c_void_p), 2) == len(full)
        assert np.array_equal(part, np.r_[full[:2], 7])
    finally:
        gg.close()
        debug_lib(capi).b200ldu_layout_debug_destroy(h)


@pytest.mark.parametrize("kind", ["P", "U"])
@pytest.mark.parametrize("dims,merge", [((9, 9, 9), 1), ((7, 5, 3), 1), ((16, 14, 12), 2)])
def test_oracle_coarse_matrix_accessor(meshmod, orc, kind, dims, merge):
    """orc_gamg_coarse_matrix level by level equals ref_ldu.coarse_matrix, the plain summation that the reference's own
    agglomeration functors reproduce (tests/test_reference_functors.py)"""
    m, c, om, og = oracle_case(meshmod, orc, kind, dims, merge)
    D, U, L = c["diag"], c["upper"], c["lower"]
    for lev in range(og.nLevels):
        Dn, Un, Ln = ref_ldu.coarse_matrix(og.restrict_addr(lev), og.face_restrict_addr(lev), og.face_flip(lev),
                                           og.ncells(lev), og.nfaces(lev), D, U, L)
        cm = og.coarse_matrix(om, lev)
        assert gl.first_difference(cm["diag"], Dn) is None, lev
        assert gl.first_difference(cm["upper"], Un) is None, lev
        assert (L is None and cm["lower"] is None) or gl.first_difference(cm["lower"], Ln) is None, lev
        D, U, L = Dn, Un, Ln


def test_scale_reorder_calibration(meshmod, orc):
    """The bound on psi of the device's scaleCorrection 1 solves (tests/test_gpu_gamg_lockstep.py) stays four times
    above what reordering the oracle's two scaling sums does to its own psi."""
    assert gl.measure_scale_reorder(orc, meshmod) <= gl.SCALE_REORDER_BOUND / 4
