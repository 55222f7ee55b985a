// fieldops_kernels.cuh -- device code of csrc/fieldops.cu, free of launch syntax (compiled for the host by
// tests/host_kernels/ as well).
#ifndef B200LDU_FIELDOPS_KERNELS_CUH
#define B200LDU_FIELDOPS_KERNELS_CUH
#include <cstddef>

namespace fieldk
{
namespace // internal linkage: the headers are included by more than one translation unit
{
enum { OP_ADD = 0, OP_SUB = 1, OP_MUL = 2, OP_DIV = 3, OP_MIN = 4, OP_MAX = 5 };
enum { UN_NEG = 0, UN_MAG = 1, UN_S_MUL = 2, UN_S_RDIV = 3, UN_S_ADD = 4, UN_S_RSUB = 5, UN_S_MIN = 6, UN_S_MAX = 7,
       UN_S_SUB = 8, UN_S_DIV = 9, UN_COPY = 10, UN_POS = 11 };
enum { LIM_UPWIND = 0, LIM_LINEAR = 1, LIM_LIMITED_LINEAR = 2, LIM_VANLEER = 3, LIM_MINMOD = 4 };

// max / min as the reference defines them for scalars (label.H:285-297, instantiated for doubles by doubleFloat.H:69-86):
// the second operand on a tie (max(+0, -0) is -0) and whenever either operand is NaN, where fmax / fmin would return the
// other operand
__device__ __forceinline__ double ref_max(double s1, double s2) { return (s1 > s2) ? s1 : s2; }
__device__ __forceinline__ double ref_min(double s1, double s2) { return (s1 < s2) ? s1 : s2; }

__device__ __forceinline__ double bin(int op, double a, double b)
{
    switch (op) {
    case OP_ADD: return __dadd_rn(a, b);
    case OP_SUB: return __dsub_rn(a, b);
    case OP_MUL: return __dmul_rn(a, b);
    case OP_DIV: return __ddiv_rn(a, b);
    case OP_MIN: return ref_min(a, b);
    default: return ref_max(a, b);
    }
}

// out[i][k] = a[i][k or 0] op b[i][k or 0]; nc = components of the result
__global__ void binary_kernel(long long n, int nc, int ncA, int ncB, int op, const double *a, const double *b, double *out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * nc) return;
    const long long e = i / nc;
    const int k = (int)(i - e * nc);
    const double x = a[ncA == 1 ? e : e * ncA + k], y = b[ncB == 1 ? e : e * ncB + k];
    out[i] = bin(op, x, y);
}

__global__ void unary_kernel(long long n, int op, double s, const double *a, double *out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double x = a[i];
    double r;
    switch (op) {
    case UN_NEG: r = -x; break;
    case UN_MAG: r = fabs(x); break;
    case UN_S_MUL: r = __dmul_rn(s, x); break;
    case UN_S_RDIV: r = __ddiv_rn(s, x); break;
    case UN_S_ADD: r = __dadd_rn(x, s); break;
    case UN_S_RSUB: r = __dsub_rn(s, x); break;
    case UN_S_MIN: r = ref_min(x, s); break;
    case UN_S_MAX: r = ref_max(x, s); break;
    case UN_S_SUB: r = __dsub_rn(x, s); break;
    case UN_S_DIV: r = __ddiv_rn(x, s); break;
    case UN_POS: r = x >= 0 ? 1.0 : 0.0; break; // pos(), Scalar.H:119-122
    default: r = x; break;
    }
    out[i] = r;
}

// Vector & Vector per element: (a.x*b.x + a.y*b.y) + a.z*b.z  (VectorI.H operator&)
__global__ void dot3_kernel(long long n, const double *__restrict__ a, const double *__restrict__ b, double *__restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double s = __dadd_rn(__dmul_rn(a[3 * i], b[3 * i]), __dmul_rn(a[3 * i + 1], b[3 * i + 1]));
    out[i] = __dadd_rn(s, __dmul_rn(a[3 * i + 2], b[3 * i + 2]));
}

// magSqr(symm(T)) per element of a tensor field (9 components, row-major T[i][j] as gauss_grad / grad_linear write it): the
// production term of the k-epsilon model, G = nut*2*magSqr(symm(fvc::grad(U))) (kEpsilon.C:235).  symm (TensorI.H:483-491):
// (xx, 0.5*(xy + yx), 0.5*(xz + zx), yy, 0.5*(yz + zy), zz); magSqr of a SymmTensor (SymmTensorI.H:276-284):
// magSqr(xx) + 2*magSqr(xy) + 2*magSqr(xz) + magSqr(yy) + 2*magSqr(yz) + magSqr(zz), added left to right
__global__ void symm_magsqr_kernel(long long n, const double *__restrict__ T, double *__restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *t = T + 9 * i;
    const double xx = t[0], yy = t[4], zz = t[8];
    const double xy = __dmul_rn(0.5, __dadd_rn(t[1], t[3])), xz = __dmul_rn(0.5, __dadd_rn(t[2], t[6])),
                 yz = __dmul_rn(0.5, __dadd_rn(t[5], t[7]));
    double s = __dmul_rn(xx, xx);
    s = __dadd_rn(s, __dmul_rn(2.0, __dmul_rn(xy, xy)));
    s = __dadd_rn(s, __dmul_rn(2.0, __dmul_rn(xz, xz)));
    s = __dadd_rn(s, __dmul_rn(yy, yy));
    s = __dadd_rn(s, __dmul_rn(2.0, __dmul_rn(yz, yz)));
    out[i] = __dadd_rn(s, __dmul_rn(zz, zz));
}

// snGradScheme::snGrad on the internal faces (snGradScheme.C:101-160): d*(vf[nei] - vf[own])
__global__ void sngrad_kernel(int nFaces, int nc, const int *__restrict__ l, const int *__restrict__ u,
                              const double *__restrict__ delta, const double *__restrict__ vf, double *__restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)nFaces * nc) return;
    const int f = (int)(i / nc), k = (int)(i - (long long)f * nc);
    out[i] = __dmul_rn(delta[f], __dsub_rn(vf[(size_t)u[f] * nc + k], vf[(size_t)l[f] * nc + k]));
}

// NVDTVD::r (limitedSchemes/LimitedScheme/NVDTVD.H:99-127): ratio of the upwind-side cell gradient (projected on
// d = C[nei] - C[own]) to the face gradient, r = 2*(gradcf/gradf) - 1, clipped when the face gradient vanishes
__device__ __forceinline__ double nvdtvd_r(double faceFlux, double phiP, double phiN, const double *gP, const double *gN,
                                           const double *d)
{
    const double gradf = __dsub_rn(phiN, phiP);
    const double *g = faceFlux > 0 ? gP : gN;
    // Vector & Vector: (d.x*g.x + d.y*g.y) + d.z*g.z (VectorI.H operator&)
    const double gradcf = __dadd_rn(__dadd_rn(__dmul_rn(d[0], g[0]), __dmul_rn(d[1], g[1])), __dmul_rn(d[2], g[2]));
    if (fabs(gradcf) >= __dmul_rn(1000.0, fabs(gradf))) {
        const double sc = gradcf >= 0 ? 1.0 : -1.0, sf = gradf >= 0 ? 1.0 : -1.0; // sign(), Scalar.H:112-116
        return __dsub_rn(__dmul_rn(__dmul_rn(2000.0, sc), sf), 1.0);               // 2*1000*sign*sign - 1
    }
    return __dsub_rn(__dmul_rn(2.0, __ddiv_rn(gradcf, gradf)), 1.0);
}

// LimitedScheme::calcLimiter on the internal faces (LimitedScheme.C:60-140) for a scalar field: limiter value per
// face from the scheme's limiter function -- upwind 0 (upwind.H:103-118), linear 1, limitedLinear
// max(min(2/max(k,SMALL)*r, 1), 0) (limitedLinear.H:64-101), vanLeer (r + |r|)/(1 + |r|) (vanLeer.H:66-85),
// Minmod max(min(r, 1), 0) (Minmod.H:66-85)
__device__ __forceinline__ double face_limiter(int scheme, double twoByk, int o, int n, double faceFlux,
                                               const double *__restrict__ vf, const double *__restrict__ gradc,
                                               const double *__restrict__ C)
{
    if (scheme == LIM_UPWIND || scheme == LIM_LINEAR) return scheme == LIM_LINEAR ? 1.0 : 0.0;
    const double d[3] = {__dsub_rn(C[3 * (size_t)n], C[3 * (size_t)o]), __dsub_rn(C[3 * (size_t)n + 1], C[3 * (size_t)o + 1]),
                         __dsub_rn(C[3 * (size_t)n + 2], C[3 * (size_t)o + 2])};
    const double r = nvdtvd_r(faceFlux, vf[o], vf[n], gradc + 3 * (size_t)o, gradc + 3 * (size_t)n, d);
    if (scheme == LIM_LIMITED_LINEAR) return fmax(fmin(__dmul_rn(twoByk, r), 1.0), 0.0);
    if (scheme == LIM_VANLEER) return __ddiv_rn(__dadd_rn(r, fabs(r)), __dadd_rn(1.0, fabs(r)));
    return fmax(fmin(r, 1.0), 0.0);
}

__global__ void limiter_kernel(int nFaces, int scheme, double twoByk, const int *__restrict__ l, const int *__restrict__ u,
                               const double *__restrict__ faceFlux, const double *__restrict__ vf,
                               const double *__restrict__ gradc, const double *__restrict__ C, double *__restrict__ out)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFaces) return;
    if (scheme == LIM_UPWIND || scheme == LIM_LINEAR) { // neither reads its arguments, which may be NULL
        out[f] = scheme == LIM_LINEAR ? 1.0 : 0.0;
        return;
    }
    out[f] = face_limiter(scheme, twoByk, l[f], u[f], faceFlux[f], vf, gradc, C);
}

// limitedSurfaceInterpolationScheme::weights (limitedSurfaceInterpolationScheme.C:155-212):
// w = limiter*cdWeight + (1 - limiter)*pos(faceFlux); without a limiter field: upwind, w = pos(faceFlux) (upwind.H:120-123)
__global__ void limited_weights_kernel(long long n, const double *__restrict__ limiter, const double *__restrict__ cd,
                                       const double *__restrict__ faceFlux, double *__restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double p = faceFlux[i] >= 0 ? 1.0 : 0.0;
    if (!limiter) {
        out[i] = p;
        return;
    }
    const double lim = limiter[i];
    out[i] = __dadd_rn(__dmul_rn(lim, cd[i]), __dmul_rn(__dsub_rn(1.0, lim), p));
}

// patchInternalField: out[i][k] = field[cells[i]][k]
__global__ void gather_kernel(int n, int nc, const int *__restrict__ cells, const double *__restrict__ f, double *__restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * nc) return;
    const int e = i / nc, k = i - e * nc;
    out[i] = f[(size_t)cells[e] * nc + k];
}
} // namespace
} // namespace fieldk
#endif
