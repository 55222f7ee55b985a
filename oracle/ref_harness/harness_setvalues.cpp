/*
 * harness_setvalues.cpp -- runs the REFERENCE'S OWN fvMatrix<scalar>::setValues on the CPU.  TEST INFRASTRUCTURE ONLY.
 * Builds on harness_fvm.cpp (the same reference sources and shims, included whole) and adds one entry point:
 *   setValues -> setValuesFromList   FV/fvMatrices/fvMatrix/fvMatrix.C:940-950, :456-657, functors :350-450
 * For a symmetric matrix the harness hands the shim's lduMatrix the copy of upper that the reference's non-const
 * lduMatrix::lower() makes on first use (lduMatrix.C:221-238), before setValues runs: setValuesFromList asks for lower()
 * (:582) before it first tests asymmetric() (:608), so the reference sees the same matrix either way.
 */
#define protected public
#define private public
#include "fvm_shim.h"
#undef protected
#undef private
#include <memory>
namespace Foam
{
// the cell and face masks of setValuesFromList are gpuList<bool>, which std::vector<bool> cannot back (no data())
template <> class gpuList<bool>
{
    std::unique_ptr<bool[]> v_;
    label n_ = 0;

public:
    typedef bool *iterator;
    typedef const bool *const_iterator;
    gpuList(label n, const bool &x) : v_(new bool[(size_t)n]), n_(n) { std::fill(v_.get(), v_.get() + n, x); }
    label size() const { return n_; }
    bool *data() { return v_.get(); }
    const bool *data() const { return v_.get(); }
    iterator begin() { return v_.get(); }
    iterator end() { return v_.get() + n_; }
    const_iterator begin() const { return v_.get(); }
    const_iterator end() const { return v_.get() + n_; }
};
} // namespace Foam
// the shim's fvMesh::boundaryMesh() is an empty stub (the other harness entry points never loop over it); setValuesFromList
// clears the patch coefficients in forAll(mesh.boundaryMesh(), patchi) (:624), over the same patches as mesh.boundary()
#define boundaryMesh boundary
#include "harness_fvm.cpp"

extern "C" {
/* nCalls successive setValues on one matrix: call j sets cells[callStart[j] .. callStart[j+1]) to values[...].  In and out:
 * psi, source [n], upper [nF], ic / bc (flat over the patches).  lower: NULL for a symmetric matrix; lowerOut receives the
 * lower coefficients afterwards.  diagOut: the diagonal afterwards.  Returns 2 when the matrix is asymmetric afterwards, 1 when
 * it is symmetric, < 0 on an error. */
int ref_fvm_set_values(int n, int nF, const int *l, const int *u, const int *ownerStart, const int *losortStart, const int *losort,
                       int nP, const int *patchStart, const int *faceCells, double *psi, const double *diag, double *upper,
                       const double *lower, double *source, double *ic, double *bc, int nCalls, const int *callStart,
                       const int *cells, const double *values, double *diagOut, double *lowerOut)
{
    try {
        const int tot = nP ? patchStart[nP] : 0;
        std::vector<int> coupled((size_t)std::max(nP, 1), 0);
        std::vector<double> zP((size_t)tot + 1, 0.0), V((size_t)n, 1.0);
        Case<scalar> C(n, nF, l, u, ownerStart, losortStart, losort, nP, patchStart, faceCells, coupled.data(), zP.data(), V.data(), psi,
                       diag, upper, lower, source, ic, bc);
        fvMatrix<scalar> &M = *C.M;
        if (!lower) M.lower() = tmp<scalargpuField>(new scalargpuField(upper, nF)); // what lduMatrix::lower() copies on first use
        for (int j = 0; j < nCalls; j++) {
            const int s = callStart[j], k = callStart[j + 1] - s;
            M.setValues(labelgpuList(cells + s, k), scalargpuField(values + s, k));
        }
        put(C.psi.internal_, psi);
        put(M.diag(), diagOut);
        put(M.upper(), upper);
        put(static_cast<const lduMatrix &>(M).lower(), lowerOut);
        put(M.source(), source);
        for (int p = 0; p < nP; p++) {
            put(M.internalCoeffs()[p], ic + patchStart[p]);
            put(M.boundaryCoeffs()[p], bc + patchStart[p]);
        }
        return M.asymmetric() ? 2 : (M.symmetric() ? 1 : 0);
    } catch (const std::exception &) {
        return -1;
    }
}
}
