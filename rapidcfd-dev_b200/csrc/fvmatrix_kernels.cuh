// fvmatrix_kernels.cuh -- device code of csrc/fvmatrix.cu (see there for the reference lines).  Kept free of launch
// syntax and runtime calls so that tests/host_kernels/ can compile the same source for the host (qualifiers and
// the rounding intrinsics defined away) and run every kernel against the oracle without a GPU.
#ifndef B200LDU_FVMATRIX_KERNELS_CUH
#define B200LDU_FVMATRIX_KERNELS_CUH
#include <cstddef>

#include "boundary_lists.cuh"

namespace fvmk
{
namespace // internal linkage: the headers are included by more than one translation unit
{
__device__ __forceinline__ double cmpt_av(const double *v, int nc) // VectorSpaceI.H:428-447: ((x + y) + z)/3
{
    if (nc == 1) return v[0];
    double s = v[0];
    for (int k = 1; k < nc; k++) s = __dadd_rn(s, v[k]);
    return __ddiv_rn(s, (double)nc);
}

// the component average of a coupled coefficient: the patch holds (c, c, c) for a vector field, and ((c + c) + c)/3 is
// not always c
__device__ __forceinline__ double coupled_av(double c, int nc)
{
    if (nc == 1) return c;
    return __ddiv_rn(__dadd_rn(__dadd_rn(c, c), c), 3.0);
}

// out[c] = in[c] + sum_b internalCoeffs(bf)[cmpt | average] + sum_coupled interfaceIntCoeffs(pf)
__global__ void boundary_diag_kernel(int nCells, BoundaryLists L, const double *__restrict__ ic, int nc, int cmpt,
                                     const double *__restrict__ couInt, const double *in, double *out)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nCells) return;
    double acc = in ? in[c] : 0.0;
    if (L.bStart)
        for (int j = L.bStart[c]; j < L.bStart[c + 1]; j++) {
            const double *v = ic + (size_t)L.bFaces[j] * nc;
            acc = __dadd_rn(acc, cmpt >= 0 ? v[cmpt] : cmpt_av(v, nc));
        }
    if (L.cStart)
        for (int j = L.cStart[c]; j < L.cStart[c + 1]; j++)
            acc = __dadd_rn(acc, cmpt >= 0 ? couInt[L.cFaces[j]] : coupled_av(couInt[L.cFaces[j]], nc));
    out[c] = acc;
}

// out[c][k] = in[c][k] + sum_b boundaryCoeffs(bf)[k] + (pnf ? sum_coupled interfaceBouCoeffs(pf)*pnf(pf)[k])
template <int NC>
__global__ void boundary_source_kernel(int nCells, BoundaryLists L, const double *__restrict__ bc,
                                       const double *__restrict__ couBou, const double *__restrict__ pnf,
                                       const double *in, double *out)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nCells) return;
    double acc[NC];
#pragma unroll
    for (int k = 0; k < NC; k++) acc[k] = in[(size_t)c * NC + k];
    if (L.bStart)
        for (int j = L.bStart[c]; j < L.bStart[c + 1]; j++) {
            const int bf = L.bFaces[j];
#pragma unroll
            for (int k = 0; k < NC; k++) acc[k] = __dadd_rn(acc[k], bc[(size_t)bf * NC + k]);
        }
    if (L.cStart && pnf)
        for (int j = L.cStart[c]; j < L.cStart[c + 1]; j++) {
            const int pf = L.cFaces[j];
            const double b = couBou[pf];
#pragma unroll
            for (int k = 0; k < NC; k++) acc[k] = __dadd_rn(acc[k], __dmul_rn(b, pnf[(size_t)pf * NC + k]));
        }
#pragma unroll
    for (int k = 0; k < NC; k++) out[(size_t)c * NC + k] = acc[k];
}

// component k of an interleaved field, minus the coupled products again when pnf is given
// (updateMatrixInterfaces on the source inside the component loop, fvMatrixSolve.C:170-186)
__global__ void component_kernel(int nCells, int nc, int k, BoundaryLists L, const double *__restrict__ couBou,
                                 const double *__restrict__ pnf, const double *__restrict__ in, double *__restrict__ out)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nCells) return;
    double acc = in[(size_t)c * nc + k];
    if (L.cStart && pnf)
        for (int j = L.cStart[c]; j < L.cStart[c + 1]; j++) {
            const int pf = L.cFaces[j];
            acc = __dsub_rn(acc, __dmul_rn(couBou[pf], pnf[(size_t)pf * nc + k]));
        }
    out[c] = acc;
}

__global__ void set_component_kernel(int nCells, int nc, int k, const double *__restrict__ in, double *__restrict__ out)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < nCells) out[(size_t)c * nc + k] = in[c];
}

// A = (diag + sum_b cmptAv(internalCoeffs) + sum_coupled interfaceIntCoeffs)/V
__global__ void A_kernel(int nCells, BoundaryLists L, const double *__restrict__ ic, int nc,
                         const double *__restrict__ couInt, const double *__restrict__ diag,
                         const double *__restrict__ V, double *__restrict__ out)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nCells) return;
    double acc = diag[c];
    if (L.bStart)
        for (int j = L.bStart[c]; j < L.bStart[c + 1]; j++)
            acc = __dadd_rn(acc, cmpt_av(ic + (size_t)L.bFaces[j] * nc, nc));
    if (L.cStart)
        for (int j = L.cStart[c]; j < L.cStart[c + 1]; j++) acc = __dadd_rn(acc, coupled_av(couInt[L.cFaces[j]], nc));
    out[c] = __ddiv_rn(acc, V[c]);
}

// H = ((lduMatrix::H(psi) + source) + boundary source)/V with lduMatrix::H = 0 - sum_own upper*psi[nei]
// - sum_nei lower*psi[own] (lduMatrixTemplates.C:50-84; products rounded, negated, added)
template <int NC>
__global__ void H_kernel(int nCells, const int *__restrict__ ownerStart, const int *__restrict__ u,
                         const int *__restrict__ losortStart, const int *__restrict__ losort, const int *__restrict__ l,
                         const double *__restrict__ upper, const double *__restrict__ lower, BoundaryLists L,
                         const double *__restrict__ bc, const double *__restrict__ couBou,
                         const double *__restrict__ pnf, const double *__restrict__ psi,
                         const double *__restrict__ source, const double *__restrict__ V, double *__restrict__ out)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nCells) return;
    // load scheduling as in fv_kernels.cuh: everything known up front first, then the first batch of coefficients and indices
    // together, then what the indices point at -- the sums keep the reference's order
    constexpr int B = 3;
    const int o0 = ownerStart[c], o1 = ownerStart[c + 1], n0 = losortStart[c], n1 = losortStart[c + 1];
    int b0 = 0, b1 = 0, c0 = 0, c1 = 0;
    if (L.bStart) b0 = L.bStart[c], b1 = L.bStart[c + 1];
    if (L.cStart && pnf) c0 = L.cStart[c], c1 = L.cStart[c + 1];
    const double v = V[c];
    double src[NC];
#pragma unroll
    for (int k = 0; k < NC; k++) src[k] = source[(size_t)c * NC + k];
    double oa[B], na[B];
    int on[B], fi[B], no[B], bf0 = 0, pf0 = 0;
#pragma unroll
    for (int b = 0; b < B; b++)
        if (o0 + b < o1) oa[b] = upper[o0 + b], on[b] = u[o0 + b];
#pragma unroll
    for (int b = 0; b < B; b++)
        if (n0 + b < n1) fi[b] = losort[n0 + b];
    if (b0 < b1) bf0 = L.bFaces[b0];
    if (c0 < c1) pf0 = L.cFaces[c0];
#pragma unroll
    for (int b = 0; b < B; b++)
        if (n0 + b < n1) na[b] = lower[fi[b]], no[b] = l[fi[b]];
    double acc[NC];
#pragma unroll
    for (int k = 0; k < NC; k++) acc[k] = 0.0;
#pragma unroll
    for (int b = 0; b < B; b++)
        if (o0 + b < o1)
#pragma unroll
            for (int k = 0; k < NC; k++) acc[k] = __dadd_rn(acc[k], -__dmul_rn(oa[b], psi[(size_t)on[b] * NC + k]));
    for (int f = o0 + B; f < o1; f++) {
        const double a = upper[f];
        const int n = u[f];
#pragma unroll
        for (int k = 0; k < NC; k++) acc[k] = __dadd_rn(acc[k], -__dmul_rn(a, psi[(size_t)n * NC + k]));
    }
#pragma unroll
    for (int b = 0; b < B; b++)
        if (n0 + b < n1)
#pragma unroll
            for (int k = 0; k < NC; k++) acc[k] = __dadd_rn(acc[k], -__dmul_rn(na[b], psi[(size_t)no[b] * NC + k]));
    for (int q = n0 + B; q < n1; q++) {
        const int f = losort[q];
        const double a = lower[f];
        const int o = l[f];
#pragma unroll
        for (int k = 0; k < NC; k++) acc[k] = __dadd_rn(acc[k], -__dmul_rn(a, psi[(size_t)o * NC + k]));
    }
#pragma unroll
    for (int k = 0; k < NC; k++) acc[k] = __dadd_rn(acc[k], src[k]);
    for (int j = b0; j < b1; j++) {
        const int bf = j == b0 ? bf0 : L.bFaces[j];
#pragma unroll
        for (int k = 0; k < NC; k++) acc[k] = __dadd_rn(acc[k], bc[(size_t)bf * NC + k]);
    }
    for (int j = c0; j < c1; j++) {
        const int pf = j == c0 ? pf0 : L.cFaces[j];
        const double b = couBou[pf];
#pragma unroll
        for (int k = 0; k < NC; k++) acc[k] = __dadd_rn(acc[k], __dmul_rn(b, pnf[(size_t)pf * NC + k]));
    }
#pragma unroll
    for (int k = 0; k < NC; k++) out[(size_t)c * NC + k] = __ddiv_rn(acc[k], v);
}

// flux: internal faces upper*psi[nei] - lower*psi[own] per component (lduMatrixTemplates.C:40-49,108-149)
template <int NC>
__global__ void flux_internal_kernel(int nFaces, const int *__restrict__ l, const int *__restrict__ u,
                                     const double *__restrict__ upper, const double *__restrict__ lower,
                                     const double *__restrict__ psi, double *__restrict__ out)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFaces) return;
    const double a = upper[f], b = lower[f];
    const int o = l[f], n = u[f];
#pragma unroll
    for (int k = 0; k < NC; k++)
        out[(size_t)f * NC + k] = __dsub_rn(__dmul_rn(a, psi[(size_t)n * NC + k]), __dmul_rn(b, psi[(size_t)o * NC + k]));
}

// boundary faces: internalCoeffs*psi[cell] - boundaryCoeffs (coupled: - boundaryCoeffs*pnf), fvMatrix.C:1622-1654
template <int NC>
__global__ void flux_boundary_kernel(int nB, const int *__restrict__ faceCells, const double *__restrict__ ic,
                                     int icStride, const double *__restrict__ bc, int bcStride,
                                     const double *__restrict__ pnf, const double *__restrict__ psi,
                                     double *__restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nB) return;
    const int c = faceCells[i];
#pragma unroll
    for (int k = 0; k < NC; k++) {
        const double a = ic[(size_t)i * icStride + (icStride == 1 ? 0 : k)];
        const double b = bc[(size_t)i * bcStride + (bcStride == 1 ? 0 : k)];
        const double nb = pnf ? __dmul_rn(b, pnf[(size_t)i * NC + k]) : b;
        out[(size_t)i * NC + k] = __dsub_rn(__dmul_rn(a, psi[(size_t)c * NC + k]), nb);
    }
}

// source - boundaryDiag*psi (fvScalarMatrixResidualFunctor, fvScalarMatrix.C:195-227)
__global__ void residual_source_kernel(int nCells, BoundaryLists L, const double *__restrict__ ic,
                                       const double *__restrict__ couInt, const double *__restrict__ psi,
                                       const double *__restrict__ source, double *__restrict__ out)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nCells) return;
    double bd = 0.0;
    if (L.bStart)
        for (int j = L.bStart[c]; j < L.bStart[c + 1]; j++) bd = __dadd_rn(bd, ic[L.bFaces[j]]);
    if (L.cStart)
        for (int j = L.cStart[c]; j < L.cStart[c + 1]; j++) bd = __dadd_rn(bd, couInt[L.cFaces[j]]);
    out[c] = __dsub_rn(source[c], __dmul_rn(bd, psi[c]));
}

// relax (fvMatrix.C:1088-1345), one pass: D0 = D; sumOff = sum |upper| (owner side) + sum |lower| (neighbour
// side) [+ |boundaryCoeffs| of coupled faces]; D += max |internalCoeffs| (coupled: component 0);
// D = max(|D|, sumOff)/alpha; D -= min internalCoeffs (coupled: component 0); S += (D - D0)*psi
template <int NC>
__global__ void relax_kernel(int nCells, const int *__restrict__ ownerStart, const int *__restrict__ losortStart,
                             const int *__restrict__ losort, const double *__restrict__ upper,
                             const double *__restrict__ lower, BoundaryLists L, const double *__restrict__ ic,
                             const double *__restrict__ couInt, const double *__restrict__ couBou, double alpha,
                             const double *__restrict__ psi, double *diag, double *source)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nCells) return;
    // load scheduling as in fv_kernels.cuh: ranges, diagonal, psi and source first; then the owner coefficients with the losort
    // indices; then the neighbour coefficients
    constexpr int B = 3;
    const int o0 = ownerStart[c], o1 = ownerStart[c + 1], n0 = losortStart[c], n1 = losortStart[c + 1];
    const double D0 = diag[c];
    double ps[NC], src[NC];
#pragma unroll
    for (int k = 0; k < NC; k++) ps[k] = psi[(size_t)c * NC + k], src[k] = source[(size_t)c * NC + k];
    double ou[B], nl[B];
    int fi[B];
#pragma unroll
    for (int b = 0; b < B; b++)
        if (o0 + b < o1) ou[b] = upper[o0 + b];
#pragma unroll
    for (int b = 0; b < B; b++)
        if (n0 + b < n1) fi[b] = losort[n0 + b];
#pragma unroll
    for (int b = 0; b < B; b++)
        if (n0 + b < n1) nl[b] = lower[fi[b]];
    double sumOff = 0.0;
#pragma unroll
    for (int b = 0; b < B; b++)
        if (o0 + b < o1) sumOff = __dadd_rn(sumOff, fabs(ou[b]));
    for (int f = o0 + B; f < o1; f++) sumOff = __dadd_rn(sumOff, fabs(upper[f]));
#pragma unroll
    for (int b = 0; b < B; b++)
        if (n0 + b < n1) sumOff = __dadd_rn(sumOff, fabs(nl[b]));
    for (int q = n0 + B; q < n1; q++) sumOff = __dadd_rn(sumOff, fabs(lower[losort[q]]));
    double D = D0;
    if (L.bStart)
        for (int j = L.bStart[c]; j < L.bStart[c + 1]; j++) {
            const double *v = ic + (size_t)L.bFaces[j] * NC;
            double m = fabs(v[0]);
#pragma unroll
            for (int k = 1; k < NC; k++) m = fmax(m, fabs(v[k]));
            D = __dadd_rn(D, m);
        }
    if (L.cStart)
        for (int j = L.cStart[c]; j < L.cStart[c + 1]; j++) {
            const int pf = L.cFaces[j];
            D = __dadd_rn(D, couInt[pf]);
            sumOff = __dadd_rn(sumOff, fabs(couBou[pf]));
        }
    D = fmax(fabs(D), sumOff);
    D = __ddiv_rn(D, alpha);
    if (L.bStart)
        for (int j = L.bStart[c]; j < L.bStart[c + 1]; j++) {
            const double *v = ic + (size_t)L.bFaces[j] * NC;
            double m = v[0];
#pragma unroll
            for (int k = 1; k < NC; k++) m = fmin(m, v[k]);
            D = __dadd_rn(D, -m);
        }
    if (L.cStart)
        for (int j = L.cStart[c]; j < L.cStart[c + 1]; j++) D = __dadd_rn(D, -couInt[L.cFaces[j]]);
    diag[c] = D;
    const double dD = __dsub_rn(D, D0);
#pragma unroll
    for (int k = 0; k < NC; k++) source[(size_t)c * NC + k] = __dadd_rn(src[k], __dmul_rn(dD, ps[k]));
}

__global__ void set_reference_kernel(int cell, int nc, double v0, double v1, double v2, double *diag, double *source)
{
    const double v[3] = {v0, v1, v2};
    const double d = diag[cell];
    for (int k = 0; k < nc; k++)
        source[(size_t)cell * nc + k] = __dadd_rn(source[(size_t)cell * nc + k], __dmul_rn(d, v[k]));
    diag[cell] = __dmul_rn(2.0, d);
}
} // namespace
} // namespace fvmk
#endif
