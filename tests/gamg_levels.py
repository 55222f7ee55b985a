"""Helpers of the GAMG level-by-level tests (tests/test_gamg_levels_cpu.py, tests/test_gpu_gamg_lockstep.py): a numpy
restatement of the coarsest-level inverse the device uploads, the coarsest matrix in the device's numbering, the exact
componentwise backward error of x = inv b, and comparisons that name the first difference."""
import math

import numpy as np

from test_gpu_step_lockstep import two_product

# Largest componentwise backward error max_i |b - A x|_i / (|A| |x| + |b|)_i of x = inv b allowed for the coarsest
# inverse, every product and sum exact.  Measured over the coarsest matrices of tests/test_gamg_levels_cpu.py (pressure
# and momentum matrices on 16x14x12 and 9^3, mergeLevels 1-3, a convection-dominated momentum matrix that pivots) with
# right-hand sides of both signs: at most 2.9e-16.
BACKWARD_ERROR_BOUND = 2e-15


def gj_inverse(A):
    """(inverse, row swaps) of the partial-pivot Gauss-Jordan inverse the GAMG solve computes on the host for its
    coarsest level (gauss_jordan_inverse in gamg.cu), statement by statement: the first row of largest magnitude in
    column k is the pivot (strict >), rows of A and of the identity swap together, the pivot row is multiplied by
    piv = 1/A[k,k], and every other row with a nonzero factor loses factor * pivot row, each product rounded before the
    subtraction (that code is built without fused multiply-adds)."""
    A = np.array(A, dtype=np.float64, copy=True)
    N = A.shape[0]
    inv = np.eye(N)
    swaps = 0
    for k in range(N):
        p, mx = k, abs(A[k, k])
        for i in range(k + 1, N):
            if abs(A[i, k]) > mx:
                mx, p = abs(A[i, k]), i
        if mx == 0.0:
            raise ZeroDivisionError("singular")
        if p != k:
            swaps += 1
            A[[k, p]] = A[[p, k]]
            inv[[k, p]] = inv[[p, k]]
        piv = 1.0 / A[k, k]
        A[k] *= piv
        inv[k] *= piv
        for i in range(N):
            if i == k:
                continue
            fct = A[i, k]
            if fct == 0.0:
                continue
            A[i] -= fct * A[k]
            inv[i] -= fct * inv[k]
    return inv, swaps


def fma(a, b, c):
    """a*b + c rounded once"""
    p, e = two_product(a, b)
    return math.fsum([float(p), float(e), float(c)])


def inverse_apply(inv, b):
    """x[i] = sum_j inv[i, j] b[j] as the coarsest solve's kernels form it: one fused multiply-add per term, ascending j,
    from zero"""
    x = np.zeros(inv.shape[0])
    for i in range(inv.shape[0]):
        s = 0.0
        for j in range(inv.shape[1]):
            s = fma(inv[i, j], b[j], s)
        x[i] = s
    return x


def banded_matrix(owner, neighbour, diag, upper, lower, perm):
    """the dense coarsest matrix in the device's numbering: row and column perm[c] for cell c"""
    n = len(diag)
    lower = upper if lower is None else lower
    A = np.zeros((n, n))
    A[perm, perm] = diag
    for f in range(len(owner)):
        o, nb = perm[owner[f]], perm[neighbour[f]]
        A[o, nb] += upper[f]
        A[nb, o] += lower[f]
    return A


def couple(A, patchStart, faceCells, bou, nbrCell, perm):
    """subtract the interface coefficients at the neighbour cell's column, patch by patch in face order, as the
    coarsest-level assembly of one rank does: A[perm[face cell], perm[neighbour cell]] -= bou"""
    for i in range(patchStart[-1]):
        A[perm[faceCells[i]], perm[nbrCell[i]]] -= bou[i]
    return A


def backward_error(A, x, b):
    """max_i |b - A x|_i / (|A| |x| + |b|)_i, the residual summed exactly (the denominator needs no such care)"""
    worst = 0.0
    for i in range(A.shape[0]):
        p, e = two_product(A[i], x)
        r = math.fsum([float(b[i])] + list(-p) + list(-e))
        den = math.fsum(list(np.abs(p)) + [abs(float(b[i]))])
        worst = max(worst, abs(r) / den if den else (0.0 if r == 0 else math.inf))
    return worst


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def first_difference(got, ref, exact_int=False):
    """None when equal (doubles bit for bit), else a one-line description of the first differing index"""
    got, ref = np.asarray(got), np.asarray(ref)
    if got.shape != ref.shape:
        return f"shape {got.shape} != {ref.shape}"
    if exact_int:
        bad = np.nonzero(got != ref)[0]
    else:
        bad = np.nonzero(bits(got).ravel() != bits(ref).ravel())[0]
    if not len(bad):
        return None
    i = int(bad[0])
    return f"{len(bad)} differ, first at {i}: {got.ravel()[i]!r} != {ref.ravel()[i]!r}"


# psi of a scaleCorrection 1 solve against the oracle's, |dpsi| / max|psi|.  The scaling adds two global sums per level
# whose order on the device differs.  The oracle's own psi with those two sums taken in descending instead of ascending
# cell order differs by up to 2.6e-14 over SCALE_CTL on the cases of scale_cases (measure_scale_reorder;
# tests/test_gamg_levels_cpu.py re-measures it and keeps it under a quarter of the bound).  The bound is 8x that.
SCALE_REORDER_BOUND = 2e-13
SCALE_CTL = [dict(maxIter=k, nPreSweeps=p, interpolateCorrection=i) for k in (1, 7, 17) for p in (0, 1) for i in (0, 1)]


def rel_diff(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def scale_cases(orc, meshmod):
    """(kind, mesh, oracle matrix, oracle hierarchy) of the scaleCorrection cases"""
    for kind in ("P", "U"):
        m = meshmod.hex_mesh(16, 14, 12)
        c = meshmod.pressure_laplacian(m) if kind == "P" else meshmod.momentum_matrix(m)
        oa = orc.Addr(m.nCells, m.lower, m.upper)
        yield kind, m, orc.Matrix(oa, c["diag"], c["upper"], c["lower"]), orc.Gamg(oa, meshmod.face_area_pair_weights(m), 10)


def measure_scale_reorder(orc, meshmod):
    """largest |dpsi| / max|psi| between the oracle's scaleCorrection 1 solves with the two sums ascending and
    descending, over the cases of test_scale_correction"""
    worst = 0.0
    for kind, m, om, og in scale_cases(orc, meshmod):
        b = meshmod.cell_field_global(m, 42)
        for kw in SCALE_CTL:
            ctl = dict(tolerance=0.0, relTol=0.0, scaleCorrection=1, **kw)
            og.set_scale_order(False)
            a, _, _ = og.solve(om, "GaussSeidel", np.zeros(m.nCells), b, **ctl)
            og.set_scale_order(True)
            d, _, _ = og.solve(om, "GaussSeidel", np.zeros(m.nCells), b, **ctl)
            og.set_scale_order(False)
            worst = max(worst, rel_diff(d, a))
    return worst
