"""GAMG agglomeration without a GPU: b200ldu_gamg_create on a host-only addressing (b200ldu_layout_debug_create)
runs the host stage alone, and its hierarchy -- level count, forward flag, level sizes and every restrict map -- is
the oracle's."""
import importlib
import types

import numpy as np
import pytest
from layout_helpers import debug_addr, debug_lib


@pytest.fixture(scope="module")
def capi():
    g = importlib.import_module("__graft_entry__")
    g.build()
    return importlib.import_module("rapidcfd-dev_b200.capi")


def _compare(capi, meshmod, orc, dims, centres=True, merge=1, forward=1):
    m = meshmod.hex_mesh(*dims)
    w = meshmod.face_area_pair_weights(m)
    og = orc.Gamg(orc.Addr(m.nCells, m.lower, m.upper), w, 10, mergeLevels=merge, forward=forward)
    h = debug_addr(capi, m, centres)
    try:
        gg = capi.GamgAgglomeration(types.SimpleNamespace(h=h, nCells=m.nCells), w, 10, mergeLevels=merge,
                                    forward=forward)
        try:
            assert gg.nLevels == og.nLevels > 0 and gg.forward == og.forward
            for lev in range(gg.nLevels):
                assert gg.level_size(lev) == (og.ncells(lev), og.nfaces(lev))
                assert np.array_equal(gg.restrict_addr(lev), og.restrict_addr(lev))
        finally:
            gg.close()
    finally:
        debug_lib(capi).b200ldu_layout_debug_destroy(h)


@pytest.mark.parametrize("dims,centres,merge", [((12, 10, 8), True, 1), ((16, 16, 16), False, 1),
                                                ((12, 10, 8), True, 2), ((16, 16, 16), True, 3),
                                                ((16, 14, 12), True, 2), ((16, 14, 12), True, 3)])
def test_host_agglomeration_identical(capi, meshmod, orc, dims, centres, merge):
    _compare(capi, meshmod, orc, dims, centres, merge)


def test_host_agglomeration_backward_start(capi, meshmod, orc):
    _compare(capi, meshmod, orc, (12, 10, 8), forward=0)


def test_host_agglomeration_refuses_patches(capi, meshmod):
    m = meshmod.hex_mesh(6, 5, 4)
    layer = np.arange(6 * 5, dtype=np.int32)  # the cells of the z = 0 layer as one coupled patch
    h = debug_addr(capi, m, patches=(np.array([0, len(layer)], np.int32), layer))
    try:
        with pytest.raises(capi.B200LduError) as e:
            capi.GamgAgglomeration(types.SimpleNamespace(h=h, nCells=m.nCells), meshmod.face_area_pair_weights(m), 10)
        assert e.value.rc == -1 and "host-only" in str(e.value)
    finally:
        debug_lib(capi).b200ldu_layout_debug_destroy(h)
