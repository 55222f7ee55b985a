/*
 * Host execution of the device code of csrc/vof.cu (vof_kernels.cuh), in the scheme of harness.cpp, which this translation unit
 * includes for its qualifier definitions, rounding intrinsics and launcher loop.  TEST INFRASTRUCTURE ONLY.
 */
#include "harness.cpp"

#include "vof_kernels.cuh"

extern "C" {
void hk_limited_flux(int nFaces, int scheme, double twoByk, const int *l, const int *u, const double *faceFlux, const double *vf,
                     const double *gradc, const double *C, const double *cd, int fluxSign, int outSign, double *out)
{
    launch(nFaces, 256, vofk::limited_flux_kernel, nFaces, scheme, twoByk, l, u, faceFlux, vf, gradc, C, cd, fluxSign, outSign, out);
}

/* b200ldu_vof_interface_flux's two kernels in its launch order */
void hk_interface_flux(const HostCase *h, const double *w, const double *gradAlpha, const double *Sf, const double *bSf,
                       const double *bSnGrad, double deltaN, const double *phi, const double *magSf, double cAlpha, double *nHatf,
                       double *nHatfB, double *phir)
{
    launch(h->nFaces, 256, vofk::interface_flux_kernel, h->nFaces, h->l, h->u, w, gradAlpha, Sf, deltaN, phi, magSf, cAlpha, nHatf,
           phir);
    launch(h->nB, 256, vofk::interface_flux_boundary_kernel, h->nB, h->bFaceCells, gradAlpha, bSf, bSnGrad, deltaN, nHatfB);
}
}
