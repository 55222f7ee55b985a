// vof_kernels.cuh -- device code of csrc/vof.cu: the face passes of the interFoam phase-fraction step, free of launch syntax so
// that tests/host_kernels/ can run it on the host against the oracle.  One thread per face, caller order; every product,
// sum, quotient and root is rounded on its own, in the order the reference's field expressions evaluate them.
#ifndef B200LDU_VOF_KERNELS_CUH
#define B200LDU_VOF_KERNELS_CUH
#include <cstddef>

#include "fieldops_kernels.cuh"
#include "fv_kernels.cuh"

namespace vofk
{
namespace
{
#ifdef __CUDACC__
__device__ __forceinline__ double sqrt_rn(double x) { return __dsqrt_rn(x); }
#else
inline double sqrt_rn(double x) { return std::sqrt(x); }
#endif

// fvc::flux(faceFlux, vf, scheme) on the internal faces (gaussConvectionScheme.C:74-84: faceFlux*interpolate(vf) with the
// scheme's weights) without the limiter, weight and face-value fields: NVDTVD::r and the limiter function
// (fieldk::face_limiter), w = lim*cd + (1 - lim)*pos(faceFlux) (limitedSurfaceInterpolationScheme.C:155-212), the one-weight
// face value w*(vf[own] - vf[nei]) + vf[nei] (surfaceInterpolationScheme.C:272-351) and the product with the flux.
// fluxSign / outSign < 0 negate the incoming flux / the result (exact), so that -fvc::flux(-phir, alpha2, scheme)
// (alphaEqn.H:92-97) is one pass.
__global__ void limited_flux_kernel(int nFaces, int scheme, double twoByk, const int *__restrict__ l, const int *__restrict__ u,
                                    const double *__restrict__ faceFlux, const double *__restrict__ vf,
                                    const double *__restrict__ gradc, const double *__restrict__ C,
                                    const double *__restrict__ cd, int fluxSign, int outSign, double *__restrict__ out)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFaces) return;
    const int o = l[f], n = u[f];
    const double flux = fluxSign < 0 ? -faceFlux[f] : faceFlux[f];
    const double lim = fieldk::face_limiter(scheme, twoByk, o, n, flux, vf, gradc, C);
    const double p = flux >= 0 ? 1.0 : 0.0;
    const double w = __dadd_rn(__dmul_rn(lim, cd[f]), __dmul_rn(__dsub_rn(1.0, lim), p));
    const double r = __dmul_rn(flux, fvk::lin_face(w, vf[o], vf[n]));
    out[f] = outSign < 0 ? -r : r;
}

// nHatfv = gradAlphaf/(mag(gradAlphaf) + deltaN) and nHatfv & Sf (interfaceProperties.C:133-145): magSqr adds the squares left
// to right (VectorSpaceI.H:336-344), the quotient is one division per component (VectorSpaceI.H:621-630), the inner product
// (x*x + y*y) + z*z (VectorI.H operator&)
__device__ __forceinline__ double nhat_flux(const double *g, const double *S, double deltaN)
{
    const double m = sqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(g[0], g[0]), __dmul_rn(g[1], g[1])), __dmul_rn(g[2], g[2])));
    const double den = __dadd_rn(m, deltaN);
    const double nx = __ddiv_rn(g[0], den), ny = __ddiv_rn(g[1], den), nz = __ddiv_rn(g[2], den);
    return __dadd_rn(__dadd_rn(__dmul_rn(nx, S[0]), __dmul_rn(ny, S[1])), __dmul_rn(nz, S[2]));
}

// internal faces: gradAlphaf = interpolate(gradAlpha) (linear), nHatf as above and, when phi is given, the compression flux
// phir = phic*nHatf with phic = cAlpha*mag(phi/magSf) (alphaEqn.H:6, :82)
__global__ void interface_flux_kernel(int nFaces, const int *__restrict__ l, const int *__restrict__ u,
                                      const double *__restrict__ w, const double *__restrict__ gradAlpha,
                                      const double *__restrict__ Sf, double deltaN, const double *__restrict__ phi,
                                      const double *__restrict__ magSf, double cAlpha, double *__restrict__ nHatf,
                                      double *__restrict__ phir)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nFaces) return;
    const size_t o = (size_t)l[f], n = (size_t)u[f];
    const double ww = w[f];
    double g[3];
#pragma unroll
    for (int k = 0; k < 3; k++) g[k] = fvk::lin_face(ww, gradAlpha[3 * o + k], gradAlpha[3 * n + k]);
    const double nf = nhat_flux(g, Sf + 3 * (size_t)f, deltaN);
    nHatf[f] = nf;
    if (phi) phir[f] = __dmul_rn(__dmul_rn(cAlpha, fabs(__ddiv_rn(phi[f], magSf[f]))), nf);
}

// non-coupled boundary faces: the boundary value of fvc::grad(alpha1) is the cell value with its normal component replaced by
// the patch's snGrad, gGradbf += n*(snGrad - (n & gGradbf)) with n = Sf/magSf (gaussGrad.C:277-303); nHatf from it as on the
// internal faces
__global__ void interface_flux_boundary_kernel(int nBFaces, const int *__restrict__ bFaceCells,
                                               const double *__restrict__ gradAlpha, const double *__restrict__ bSf,
                                               const double *__restrict__ bSnGrad, double deltaN,
                                               double *__restrict__ nHatfB)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nBFaces) return;
    const double *S = bSf + 3 * (size_t)i, *gc = gradAlpha + 3 * (size_t)bFaceCells[i];
    const double magS = sqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(S[0], S[0]), __dmul_rn(S[1], S[1])), __dmul_rn(S[2], S[2])));
    const double nv[3] = {__ddiv_rn(S[0], magS), __ddiv_rn(S[1], magS), __ddiv_rn(S[2], magS)};
    const double ng = __dadd_rn(__dadd_rn(__dmul_rn(nv[0], gc[0]), __dmul_rn(nv[1], gc[1])), __dmul_rn(nv[2], gc[2]));
    const double s = __dsub_rn(bSnGrad[i], ng);
    double g[3];
#pragma unroll
    for (int k = 0; k < 3; k++) g[k] = __dadd_rn(gc[k], __dmul_rn(nv[k], s));
    nHatfB[i] = nhat_flux(g, S, deltaN);
}
} // namespace
} // namespace vofk
#endif
