"""The ragged and degenerate meshes of tests/hygiene_cases.py without a GPU: the oracle on every shape against dense numpy, the
host-only banded layout of every shape (b200ldu_layout_debug_*), and a dry run of tests/test_gpu_memory_hygiene.py's own logic --
the guarded-buffer helper against kernels that are wrong in the ways it exists to catch, and the field-operator references against
tests/oracle_backend.py."""
import importlib

import numpy as np
import pytest

import hygiene_cases as hc
import test_gpu_memory_hygiene as H
from layout_helpers import debug_layout
from test_layout_cpu import _check_layout


def _dense(box, coeffs, transpose=False):
    """the dense matrix Amul applies, or the one Tmul applies: the transposed face coefficients and interfaceIntCoeffs"""
    diag, upper, lower, bou, itc = coeffs
    A = np.diag(diag).astype(float)
    lower = upper if lower is None else lower
    for f in range(box.nFaces):
        A[box.lower[f], box.upper[f]] += upper[f]
        A[box.upper[f], box.lower[f]] += lower[f]
    if transpose:
        A = A.T.copy()
    _, fc, _, partner = box.coupled_arrays()
    if fc is not None:                        # result[cell] -= coeff*psi[partner]
        for i, c in enumerate(fc):
            A[c, partner[i]] -= (itc if transpose else bou)[i]
    return A


@pytest.mark.parametrize("name", hc.NAMES)
def test_shapes_and_the_oracle(orc, name):
    box = hc.build(name)
    n = box.nCells
    assert box.nFaces == 0 if name == "cell1" else box.nFaces > 0
    if name.startswith("chain"):
        assert n == int(name[5:]) and box.nFaces == n - 1
    if name.startswith("hub"):
        k = int(name[3:])
        assert np.bincount(box.lower, minlength=n)[0] == k
    if name in hc.BOXES:
        assert abs(n % 64 - 32) == 31
    if name == "isolated":
        touched = np.union1d(box.lower, box.upper)
        assert n - len(touched) > n // 2
    rng = np.random.default_rng(1)
    x, b = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    for symmetric in (True, False):
        coeffs = hc.coefficients(box, symmetric, 3)
        _, om = hc.oracle_matrix(orc, box, coeffs)
        A = _dense(box, coeffs)
        np.testing.assert_allclose(om.amul(x), A @ x, rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(om.tmul(x), _dense(box, coeffs, True) @ x, rtol=1e-13, atol=1e-13)
        solver, pre = ("PCG", "DIC") if symmetric else ("PBiCGStab", "DILU")
        psi, perf, _ = om.solve(solver, pre, np.zeros(n), b, tolerance=1e-12, maxIter=1000)
        assert perf.converged, (name, symmetric)
        np.testing.assert_allclose(psi, np.linalg.solve(A, b), rtol=0, atol=1e-9)


@pytest.mark.parametrize("band", H.BANDS)
@pytest.mark.parametrize("name", hc.NAMES)
def test_layout_of_every_shape(name, band):
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    box = hc.build(name)
    lay = debug_layout(capi, box, True, band)
    _check_layout(box, lay)
    nPad, nBands, bandRows = (int(v) for v in lay["dims"][:3])
    assert nPad >= box.nCells and nPad - box.nCells < bandRows and nBands == nPad // bandRows
    assert len(lay["sliceStart"]) == nPad // 64 + 1
    if band:
        assert bandRows == band
    if name.startswith("hub"):        # the hub's row holds every one of its faces: its slice is that wide
        assert lay["sliceW"].max() >= int(name[3:])


# ---- dry run of the GPU module's own logic -------------------------------------------------------------------------------
def _as_storage(torch, view, n):
    """n doubles from where `view` starts, reading past its end into the buffer around it (what a kernel with a wrong bound does)"""
    return torch.as_strided(view, (n,), (1,))


def test_guard_helper_catches_what_it_exists_for():
    torch = pytest.importorskip("torch")
    dev = torch.device("cpu")
    x = np.arange(1.0, 8.0)
    n = len(x)

    def right(v):
        v["y"].copy_(2 * v["x"])
    got = H.call(torch, dev, right, {"x": x}, {"y": n})
    assert np.array_equal(got["y"], 2 * x)

    def skips_last(v):
        v["y"][:-1].copy_(2 * v["x"][:-1])

    def writes_past_end(v):
        _as_storage(torch, v["y"], n + 1).copy_(torch.ones(n + 1))

    def reads_past_end(v):
        v["y"].copy_(_as_storage(torch, v["x"], n + 1)[1:])

    def writes_input(v):
        v["x"][0] = 0.0
        v["y"].copy_(v["x"])

    def writes_outside_range(v):
        v["y"].copy_(v["x"])
    for fn, msg in ((skips_last, "never written"), (writes_past_end, "guard"), (reads_past_end, "different results"),
                    (writes_input, "input was written")):
        with pytest.raises(AssertionError, match=msg):
            H.call(torch, dev, fn, {"x": x}, {"y": n})
    with pytest.raises(AssertionError, match="written outside"):
        H.call(torch, dev, writes_outside_range, {"x": x}, {"y": (n, 0, n - 2)})
    # in place: the untouched tail of an in-out array is part of the result; n = 0 works
    got = H.call(torch, dev, lambda v: v["p"][:3].mul_(2), (), (), {"p": x})
    assert np.array_equal(got["p"], np.concatenate([2 * x[:3], x[3:]]))
    got = H.call(torch, dev, lambda v: None, {"x": np.zeros(0)}, {"y": 0})
    assert got["y"].shape == (0,)
    H.same({"a": (1.0, None, np.array([0.0]))}, {"a": (1.0, None, np.array([0.0]))})
    with pytest.raises(AssertionError):
        H.same({"a": np.array([0.0])}, {"a": np.array([-0.0])})


def test_field_references_over_the_oracle_stand_in(monkeypatch):
    """the numpy references of test_gpu_memory_hygiene.test_field_operators against tests/oracle_backend.FieldOps"""
    import oracle_backend
    torch = pytest.importorskip("torch")
    monkeypatch.setenv("B200LDU_DRYRUN_ORACLE", "1")
    capi, ctx, _ = oracle_backend.fixture()
    ops = capi.FieldOps(ctx)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    for n in H.FIELD_N:
        I = H.field_inputs(n)
        for op, f in enumerate((ops.add, ops.sub, ops.mul, ops.div)):
            for nca, ncb in H.NC_MIX:
                want = f(t(I[f"a{nca}"]), t(I[f"b{ncb}"]), nca, ncb).numpy()
                assert np.array_equal(H.bits(H.binary_reference(op, I[f"a{nca}"], I[f"b{ncb}"], nca, ncb)), H.bits(want)), (n, op)
        assert np.array_equal(H.binary_reference(5, I["a1"], I["b1"], 1, 1), ops.bmax(t(I["a1"]), t(I["b1"])).numpy())
        a, s = t(I["a3"]), -1.25
        with np.errstate(divide="ignore"):
            stand_in = {0: ops.neg(a), 1: ops.mag(a), 2: ops.smul(s, a), 3: ops.rdiv(s, a), 4: ops.sadd(a, s), 5: ops.rsub(s, a),
                        6: ops.smin(a, s), 7: ops.smax(a, s), 9: ops.sdiv(a, s), 11: ops.pos(a)}
        for op, want in stand_in.items():
            assert np.array_equal(H.bits(H.unary_reference(op, I["a3"], s)), H.bits(want.numpy())), (n, op)
        assert np.array_equal(H.unary_reference(8, I["a3"], s), I["a3"] - s)
        assert np.array_equal(H.bits(H.unary_reference(10, I["a3"], s)), H.bits(I["a3"]))
        assert np.array_equal(ops.gather(torch.from_numpy(I["cells"]), t(I["a3"]), 3).numpy(), I["a3"].reshape(-1, 3)[I["cells"]].ravel())
