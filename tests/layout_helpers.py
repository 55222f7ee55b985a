"""Reader of the host-only banded layout (b200ldu_layout_debug_*) for the CPU layout tests: builds the layout of a
mesh without a GPU and returns every array the library exposes, by name."""
import ctypes as C
import os

import numpy as np

# b200ldu_layout_debug_get's `what` codes, in order (layout.cu)
WHAT = [("perm", np.int32), ("iperm", np.int32), ("sliceStart", np.int64), ("sliceW", np.uint16),
        ("sliceWL", np.uint16), ("col", np.uint16), ("code", np.int32), ("haloStart", np.int32),
        ("haloIdx", np.int32), ("dims", np.int32), ("fsSlice", np.int32), ("fsCT", np.uint32),
        ("fsCode", np.int32), ("fsListStart", np.int32), ("fsListIfc", np.int32), ("fsDims", np.int64)]


def debug_lib(capi):
    """The library with the b200ldu_layout_debug_* signatures declared."""
    L = capi.lib()
    L.b200ldu_layout_debug_get.restype = C.c_longlong
    L.b200ldu_layout_debug_get.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong]
    L.b200ldu_layout_debug_create.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
    L.b200ldu_layout_debug_destroy.argtypes = [C.c_void_p]
    return L


def debug_addr(capi, mesh, centres=True, band=None, patches=None):
    """Handle of the host-only addressing of `mesh` (its own coupled patches unless `patches` = (patchStart,
    faceCells)), built with B200LDU_BAND_ROWS=band, or without the variable when band is None.  The caller frees it
    with b200ldu_layout_debug_destroy."""
    L = debug_lib(capi)
    ps, fc = patches if patches is not None else mesh.patch_start_facecells()
    ps, fc = np.ascontiguousarray(ps, np.int32), np.ascontiguousarray(fc, np.int32)
    nP = len(ps) - 1
    l = np.ascontiguousarray(mesh.lower, np.int32)
    u = np.ascontiguousarray(mesh.upper, np.int32)
    cc = np.ascontiguousarray(mesh.cell_centres()) if centres else None
    h = C.c_void_p()
    old = os.environ.pop("B200LDU_BAND_ROWS", None)
    if band:
        os.environ["B200LDU_BAND_ROWS"] = str(band)
    try:
        rc = L.b200ldu_layout_debug_create(mesh.nCells, mesh.nFaces, l.ctypes.data, u.ctypes.data, nP,
                                           ps.ctypes.data if nP else None, fc.ctypes.data if nP else None,
                                           cc.ctypes.data if cc is not None else None, C.byref(h))
    finally:
        os.environ.pop("B200LDU_BAND_ROWS", None)
        if old is not None:
            os.environ["B200LDU_BAND_ROWS"] = old
    assert rc == 0, L.b200ldu_last_error()
    return h


def debug_layout(capi, mesh, centres=True, band=None, patches=None):
    """{name: array} of the layout of `mesh`, arguments as debug_addr."""
    L = debug_lib(capi)
    h = debug_addr(capi, mesh, centres, band, patches)
    out = {}
    for what, (name, dt) in enumerate(WHAT):
        n = L.b200ldu_layout_debug_get(h, what, None, 0)
        a = np.zeros(max(n, 1), dtype=dt)
        L.b200ldu_layout_debug_get(h, what, a.ctypes.data, n)
        out[name] = a[:n]
    L.b200ldu_layout_debug_destroy(h)
    return out
