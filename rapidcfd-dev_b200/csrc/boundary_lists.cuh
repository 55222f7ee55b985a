// boundary_lists.cuh -- the per-cell boundary-face lists the finite-volume kernels walk: taken by the kernels of
// fvmatrix_kernels.cuh, built from an addressing by boundary_lists() (internal.h).  Plain C++, so that
// tests/host_kernels/ compiles it for the host with the kernels.
#ifndef B200LDU_BOUNDARY_LISTS_CUH
#define B200LDU_BOUNDARY_LISTS_CUH

namespace fvmk
{
namespace // internal linkage: the headers are included by more than one translation unit
{
struct BoundaryLists { // per-cell CSR over the non-coupled boundary faces and over the coupled patch faces
    const int *bStart, *bFaces, *cStart, *cFaces;
};
} // namespace
} // namespace fvmk
#endif
