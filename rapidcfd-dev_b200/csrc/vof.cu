// vof.cu -- the face passes of the interFoam phase-fraction step (caller-order fields, one thread per face; device code in
// vof_kernels.cuh).
//
// Reference: applications/solvers/multiphase/interFoam/alphaEqn.H:6,82-98 (phic, phir and the three fvc::flux of a limited
// scheme), src/transportModels/interfaceProperties/interfaceProperties.C:118-159 (calculateK: nHatfv, nHatf),
// FV/finiteVolume/convectionSchemes/gaussConvectionScheme/gaussConvectionScheme.C:74-84 (flux),
// FV/interpolation/surfaceInterpolation/limitedSchemes/limitedSurfaceInterpolationScheme/limitedSurfaceInterpolationScheme.C:155-212,
// FV/finiteVolume/gradSchemes/gaussGrad/gaussGrad.C:277-303 (boundary values of fvc::grad).
#include "internal.h"

#include "vof_kernels.cuh"

using namespace vofk;

extern "C" int b200ldu_fv_limited_flux(b200ldu_addr *a, const char *scheme, double k, const double *faceFlux_d,
                                       const double *vf_d, const double *gradc_d, const double *C_d,
                                       const double *cdWeights_d, int fluxSign, int outSign, double *flux_d)
{
    if (!a || !scheme || !faceFlux_d || !vf_d || !flux_d) return B200LDU_EINVAL;
    if ((fluxSign != 1 && fluxSign != -1) || (outSign != 1 && outSign != -1)) return B200LDU_EINVAL;
    int sch;
    double twoByk;
    TRY(limiter_scheme(scheme, k, &sch, &twoByk));
    if (sch >= fieldk::LIM_LIMITED_LINEAR && (!gradc_d || !C_d)) return B200LDU_EINVAL;
    if (!cdWeights_d) return B200LDU_EINVAL;
    CUDA_TRY(cudaSetDevice(a->ctx->device));
    return launch(a->ctx, limited_flux_kernel, a->nFaces, 256, a->nFaces, sch, twoByk, a->d_l, a->d_u, faceFlux_d, vf_d, gradc_d,
                  C_d, cdWeights_d, fluxSign, outSign, flux_d);
}

extern "C" int b200ldu_vof_interface_flux(b200ldu_addr *a, const double *w_d, const double *gradAlpha_d, const double *Sf_d,
                                          const double *bSf_d, const double *bSnGrad_d, double deltaN, const double *phi_d,
                                          const double *magSf_d, double cAlpha, double *nHatf_d, double *nHatfB_d,
                                          double *phir_d)
{
    if (!a || !w_d || !gradAlpha_d || !Sf_d || !nHatf_d) return B200LDU_EINVAL;
    if (a->nBFaces && (!bSf_d || !bSnGrad_d || !nHatfB_d)) return B200LDU_EINVAL;
    if (phi_d && (!magSf_d || !phir_d)) return B200LDU_EINVAL;
    CUDA_TRY(cudaSetDevice(a->ctx->device));
    TRY(launch(a->ctx, interface_flux_kernel, a->nFaces, 256, a->nFaces, a->d_l, a->d_u, w_d, gradAlpha_d, Sf_d, deltaN, phi_d,
               magSf_d, cAlpha, nHatf_d, phir_d));
    return launch(a->ctx, interface_flux_boundary_kernel, a->nBFaces, 256, a->nBFaces, a->d_bFaceCells, gradAlpha_d, bSf_d,
                  bSnGrad_d, deltaN, nHatfB_d);
}
