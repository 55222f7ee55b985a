/*
 * ldu_oracle.c -- CPU restatement of the RapidCFD-dev lduMatrix solver core.
 * TEST INFRASTRUCTURE ONLY (see ldu_oracle.h for what is pinned to the reference's own code).
 *
 * Paths cited below are relative to /root/reference/src/OpenFOAM/matrices/lduMatrix/
 * (abbreviated LDU/) unless they start with another top-level directory.
 */
#include "ldu_oracle_internal.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* constants: LduMatrix/LduMatrix/SolverPerformance.H:269-275 */
static const double ORC_GREAT = 1e20;
static const double ORC_SMALL = 1e-20;
static const double ORC_VSMALL = 1e-300;

void orc_controls_default(orc_controls *c)
{
    memset(c, 0, sizeof(*c));
    c->tolerance = 1e-6; /* LDU/lduMatrix/lduMatrixSolver.C:167-173 */
    c->relTol = 0;
    c->maxIter = 1000;
    c->minIter = 0;
    c->nSweeps = 1;  /* LDU/solvers/smoothSolver/smoothSolver.C:80 */
    c->omega = 0.9;  /* LDU/smoothers/Jacobi/JacobiSmoother.C:34 */
    c->bicgstabRefQuirk = 0;
    /* LDU/solvers/GAMG/GAMGSolver.C:67-77 */
    c->nCellsInCoarsestLevel = 10;
    c->mergeLevels = 1;
    c->nPreSweeps = 0;
    c->preSweepsLevelMultiplier = 1;
    c->maxPreSweeps = 4;
    c->nPostSweeps = 2;
    c->postSweepsLevelMultiplier = 1;
    c->maxPostSweeps = 4;
    c->nFinestSweeps = 2;
    c->interpolateCorrection = 0;
    c->scaleCorrection = -1;
    c->directSolveCoarsest = 1;
}

/* ------------------------------------------------------------------------- */
/* addressing: LDU/lduAddressing/lduAddressing.C                              */
/* ------------------------------------------------------------------------- */

orc_addr *orc_addr_create(int nCells, int nFaces, const int *l, const int *u, int nPatches,
                          const int *patchStart, const int *faceCells)
{
    orc_addr *a = (orc_addr *)calloc(1, sizeof(orc_addr));
    a->nCells = nCells;
    a->nFaces = nFaces;
    a->l = (int *)malloc(sizeof(int) * (size_t)(nFaces > 0 ? nFaces : 1));
    a->u = (int *)malloc(sizeof(int) * (size_t)(nFaces > 0 ? nFaces : 1));
    memcpy(a->l, l, sizeof(int) * (size_t)nFaces);
    memcpy(a->u, u, sizeof(int) * (size_t)nFaces);

    /* ownerStart: row pointer over the owner-sorted face list (:202-267). Faces
     * arrive sorted by owner, so counting is enough. */
    a->ownerStart = (int *)calloc((size_t)nCells + 1, sizeof(int));
    for (int f = 0; f < nFaces; f++) a->ownerStart[l[f] + 1]++;
    for (int c = 0; c < nCells; c++) a->ownerStart[c + 1] += a->ownerStart[c];

    /* losort: stable sort of face indices by neighbour (:169-199);
     * losortStart: row pointer over that list (:270-344). Counting sort = stable. */
    a->losortStart = (int *)calloc((size_t)nCells + 1, sizeof(int));
    a->losort = (int *)malloc(sizeof(int) * (size_t)(nFaces > 0 ? nFaces : 1));
    for (int f = 0; f < nFaces; f++) a->losortStart[u[f] + 1]++;
    for (int c = 0; c < nCells; c++) a->losortStart[c + 1] += a->losortStart[c];
    {
        int *cur = (int *)malloc(sizeof(int) * ((size_t)nCells + 1));
        memcpy(cur, a->losortStart, sizeof(int) * ((size_t)nCells + 1));
        for (int f = 0; f < nFaces; f++) a->losort[cur[u[f]]++] = f;
        free(cur);
    }

    a->nPatches = nPatches;
    a->patchStart = (int *)calloc((size_t)nPatches + 1, sizeof(int));
    int tot = 0;
    if (nPatches > 0) {
        memcpy(a->patchStart, patchStart, sizeof(int) * ((size_t)nPatches + 1));
        tot = patchStart[nPatches];
    }
    a->faceCells = (int *)malloc(sizeof(int) * (size_t)(tot > 0 ? tot : 1));
    if (tot > 0) memcpy(a->faceCells, faceCells, sizeof(int) * (size_t)tot);
    return a;
}

void orc_addr_free(orc_addr *a)
{
    if (!a) return;
    free(a->l);
    free(a->u);
    free(a->ownerStart);
    free(a->losort);
    free(a->losortStart);
    free(a->patchStart);
    free(a->faceCells);
    free(a->neighbRank);
    free(a);
}

void orc_addr_set_neighb_ranks(orc_addr *a, const int *neighbRank)
{
    free(a->neighbRank);
    a->neighbRank = (int *)malloc(sizeof(int) * (size_t)(a->nPatches > 0 ? a->nPatches : 1));
    memcpy(a->neighbRank, neighbRank, sizeof(int) * (size_t)a->nPatches);
}

const int *orc_addr_owner_start(const orc_addr *a) { return a->ownerStart; }
const int *orc_addr_losort(const orc_addr *a) { return a->losort; }
const int *orc_addr_losort_start(const orc_addr *a) { return a->losortStart; }

orc_matrix *orc_matrix_create(const orc_addr *a, const double *diag, const double *upper,
                              const double *lower, const double *bouCoeffs,
                              const double *intCoeffs)
{
    orc_matrix *m = (orc_matrix *)calloc(1, sizeof(orc_matrix));
    m->a = a;
    m->diag = diag;
    m->upper = upper;
    m->lower = lower ? lower : upper; /* lduMatrix.C:328-345: lower() aliases upper() */
    m->symmetric = (lower == NULL);
    m->bou = bouCoeffs;
    m->intc = intCoeffs;
    return m;
}

void orc_matrix_free(orc_matrix *m) { free(m); }

/* ------------------------------------------------------------------------- */
/* halo helper: LDU/lduMatrix/lduMatrixUpdateMatrixInterfaces.C:30-276 +      */
/* finiteVolume/fields/fvPatchFields/constraint/processor/                    */
/* processorFvPatchScalarField.C:37-172                                       */
/* ------------------------------------------------------------------------- */

double *orc_halo_exchange(const orc_addr *a, const double *psi, const orc_comm *comm)
{
    int tot = a->nPatches ? a->patchStart[a->nPatches] : 0;
    if (tot == 0) return NULL;
    double *send = (double *)malloc(sizeof(double) * (size_t)tot);
    double *recv = (double *)calloc((size_t)tot, sizeof(double));
    for (int i = 0; i < tot; i++) send[i] = psi[a->faceCells[i]]; /* patchInternalField */
    if (comm && comm->halo) comm->halo(comm->ctx, send, recv, tot, a->nPatches, a->patchStart);
    /* cyclic patches (neighbRank[p] = -(q+1): partner patch q of this addressing): the neighbour
     * values are psi at the partner's face cells, cyclicFvPatchField.C:212-231 -- scalars are
     * not transformed */
    if (a->neighbRank)
        for (int p = 0; p < a->nPatches; p++) {
            if (a->neighbRank[p] >= 0) continue;
            int q = -a->neighbRank[p] - 1;
            int n = a->patchStart[p + 1] - a->patchStart[p];
            for (int i = 0; i < n; i++) recv[a->patchStart[p] + i] = send[a->patchStart[q] + i];
        }
    free(send);
    return recv;
}

/* reduce(v, sumOp) over the ranks, for tests that compose the oracle from Python */
void orc_comm_sum(const orc_comm *comm, double *vals, int n)
{
    if (comm && comm->sum) comm->sum(comm->ctx, vals, n);
}

/* coupledFvPatchField::patchNeighbourField for every coupled patch face (tests, fvMatrix glue) */
void orc_patch_neighbour_field(const orc_addr *a, const double *psi, const orc_comm *comm, double *out)
{
    int tot = a->nPatches ? a->patchStart[a->nPatches] : 0;
    double *pnf = orc_halo_exchange(a, psi, comm);
    for (int i = 0; i < tot; i++) out[i] = pnf[i];
    free(pnf);
}

/* result[faceCell] -= coeff*pnf (negate=false) or += (negate=true):
 * lduAddressingFunctors.H:237-262, coupledFvPatchField.C:221-257. The product is
 * rounded, its sign flipped, then added. */
static void orc_apply_interfaces(const orc_addr *a, const double *coeffs, const double *pnf,
                                 double *result, int negate)
{
    int tot = a->nPatches ? a->patchStart[a->nPatches] : 0;
    for (int i = 0; i < tot; i++) {
        double v = coeffs[i] * pnf[i];
        result[a->faceCells[i]] = result[a->faceCells[i]] + (negate ? v : -v);
    }
}

/* ------------------------------------------------------------------------- */
/* Amul / Tmul: LDU/lduMatrix/lduMatrixATmul.C:42-138 (functor), :183-342      */
/* ------------------------------------------------------------------------- */

static inline double orc_row_sum(const orc_addr *a, int c, double init, const double *U,
                                 const double *L, const double *x)
{
    /* Summation order of matrixMultiplyFunctor (:78-137): init, owner-side products
     * in face order, neighbour-side products in losort order.  (The reference adds
     * the first three of each side before any fourth owner-side term; rows with more
     * than three faces on one side therefore differ from it in association only --
     * never on hex meshes.) */
    double out = init;
    for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++) {
        double p = U[f] * x[a->u[f]];
        out = out + p;
    }
    for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++) {
        int f = a->losort[k];
        double p = L[f] * x[a->l[f]];
        out = out + p;
    }
    return out;
}

static void orc_mul_impl(const orc_matrix *m, const double *U, const double *L,
                         const double *ifc, const double *psi, double *out,
                         const orc_comm *comm)
{
    const orc_addr *a = m->a;
    double *pnf = orc_halo_exchange(a, psi, comm); /* initMatrixInterfaces :209 */
    for (int c = 0; c < a->nCells; c++) {
        double d = m->diag[c] * psi[c];
        out[c] = orc_row_sum(a, c, d, U, L, psi);
    }
    if (pnf) { /* updateMatrixInterfaces :251 */
        orc_apply_interfaces(a, ifc, pnf, out, 0);
        free(pnf);
    }
}

void orc_amul(const orc_matrix *m, const double *psi, double *Apsi, const orc_comm *comm)
{
    orc_mul_impl(m, m->upper, m->lower, m->bou, psi, Apsi, comm);
}

/* Tmul swaps upper/lower and uses interfaceIntCoeffs (:264-342; PBiCG.C:96) */
void orc_tmul(const orc_matrix *m, const double *psi, double *Tpsi, const orc_comm *comm)
{
    orc_mul_impl(m, m->lower, m->upper, m->intc, psi, Tpsi, comm);
}

/* sumA: lduMatrixATmul.C:345-395 */
void orc_sumA(const orc_matrix *m, double *sumA)
{
    const orc_addr *a = m->a;
    for (int c = 0; c < a->nCells; c++) {
        double out = m->diag[c];
        for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++) out = out + m->upper[f];
        for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++)
            out = out + m->lower[a->losort[k]];
        sumA[c] = out;
    }
    int tot = a->nPatches ? a->patchStart[a->nPatches] : 0;
    for (int i = 0; i < tot; i++) /* :374-393: minus interface boundary coeffs */
        sumA[a->faceCells[i]] = sumA[a->faceCells[i]] + (-m->bou[i]);
}

/* residual: lduMatrixATmul.C:397-496; rA = source - diag*psi - sum(off-diag) with the
 * interface term entering with flipped sign (:455-463) */
void orc_residual(const orc_matrix *m, const double *psi, const double *source, double *rA,
                  const orc_comm *comm)
{
    const orc_addr *a = m->a;
    double *pnf = orc_halo_exchange(a, psi, comm);
    for (int c = 0; c < a->nCells; c++) {
        double out = source[c] - m->diag[c] * psi[c]; /* lduMatrixDiagonalResidualFunctor */
        for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++) {
            double p = m->upper[f] * psi[a->u[f]];
            out = out + (-p);
        }
        for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++) {
            int f = a->losort[k];
            double p = m->lower[f] * psi[a->l[f]];
            out = out + (-p);
        }
        rA[c] = out;
    }
    if (pnf) {
        int tot = a->patchStart[a->nPatches];
        for (int i = 0; i < tot; i++) { /* coeff = -bou, contribution = -(coeff*pnf) */
            double v = (-m->bou[i]) * pnf[i];
            rA[a->faceCells[i]] = rA[a->faceCells[i]] + (-v);
        }
        free(pnf);
    }
}

/* H: lduMatrixOperations.C:107-155 ; Hpsi = -(U psi(nei) + L psi(own)) */
void orc_H(const orc_matrix *m, const double *psi, double *Hpsi)
{
    const orc_addr *a = m->a;
    for (int c = 0; c < a->nCells; c++) {
        double out = 0.0;
        for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++) {
            double p = m->upper[f] * psi[a->u[f]];
            out = out + (-p);
        }
        for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++) {
            int f = a->losort[k];
            double p = m->lower[f] * psi[a->l[f]];
            out = out + (-p);
        }
        Hpsi[c] = out;
    }
}

/* H1: lduMatrixATmul.C:515-554 ; H1 = -(sum upper + sum lower) per row */
void orc_H1(const orc_matrix *m, double *H1)
{
    const orc_addr *a = m->a;
    for (int c = 0; c < a->nCells; c++) {
        double out = 0.0;
        for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++) out = out + (-m->upper[f]);
        for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++)
            out = out + (-m->lower[a->losort[k]]);
        H1[c] = out;
    }
}

/* faceH: lduMatrixTemplates.C:40-49,108-149 ; upper*psi[u] - lower*psi[l] per face */
void orc_faceH(const orc_matrix *m, const double *psi, double *faceHpsi)
{
    const orc_addr *a = m->a;
    for (int f = 0; f < a->nFaces; f++) {
        double p1 = m->upper[f] * psi[a->u[f]];
        double p2 = m->lower[f] * psi[a->l[f]];
        faceHpsi[f] = p1 - p2;
    }
}

/* sumDiag / negSumDiag / sumMagOffDiag: lduMatrixOperations.C:36-104.  The row
 * receives lower[f] for faces it owns and upper[f] for faces where it is neighbour. */
void orc_sumDiag(const orc_addr *a, const double *upper, const double *lower, double *diag)
{
    if (!lower) lower = upper;
    for (int c = 0; c < a->nCells; c++) {
        double out = diag[c];
        for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++) out = out + lower[f];
        for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++)
            out = out + upper[a->losort[k]];
        diag[c] = out;
    }
}

void orc_negSumDiag(const orc_addr *a, const double *upper, const double *lower, double *diag)
{
    if (!lower) lower = upper;
    for (int c = 0; c < a->nCells; c++) {
        double out = diag[c];
        for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++) out = out - lower[f];
        for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++)
            out = out - upper[a->losort[k]];
        diag[c] = out;
    }
}

void orc_sumMagOffDiag(const orc_addr *a, const double *upper, const double *lower, double *out_)
{
    if (!lower) lower = upper;
    for (int c = 0; c < a->nCells; c++) {
        double out = out_[c];
        for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++) out = out + fabs(upper[f]);
        for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++)
            out = out + fabs(lower[a->losort[k]]);
        out_[c] = out;
    }
}

/* ------------------------------------------------------------------------- */
/* global reductions: fields/Fields/gpuField/gpuFieldCommonFunctions.C:420-636 */
/* (thrust::reduce order is unspecified; the oracle sums in index order)        */
/* ------------------------------------------------------------------------- */

double orc_gsum(const double *x, int n, const orc_comm *comm)
{
    double s = 0;
    for (int i = 0; i < n; i++) s += x[i];
    if (comm && comm->sum) comm->sum(comm->ctx, &s, 1);
    return s;
}

double orc_gsumprod(const double *x, const double *y, int n, const orc_comm *comm)
{
    double s = 0;
    for (int i = 0; i < n; i++) s += x[i] * y[i];
    if (comm && comm->sum) comm->sum(comm->ctx, &s, 1);
    return s;
}

double orc_gsummag(const double *x, int n, const orc_comm *comm)
{
    double s = 0;
    for (int i = 0; i < n; i++) s += fabs(x[i]);
    if (comm && comm->sum) comm->sum(comm->ctx, &s, 1);
    return s;
}

/* the lockstep hook (ldu_oracle.h): per thread, so concurrent tests do not see each other's */
static _Thread_local orc_reduce_fn hookFn;
static _Thread_local void *hookCtx;
static _Thread_local int stagedAinv;

void orc_set_reduce_hook(orc_reduce_fn fn, void *ctx)
{
    hookFn = fn;
    hookCtx = ctx;
}

void orc_set_staged_ainv(int on) { stagedAinv = on; }

/* a global sum at a named call site: the oracle's own value, or the hook's when it is armed */
static double site_sum(int site, int iter, int op, const double *x, const double *y, int n, const orc_comm *comm)
{
    double s = op == ORC_RED_PROD ? orc_gsumprod(x, y, n, comm) : op == ORC_RED_MAG ? orc_gsummag(x, n, comm)
                                                                                 : orc_gsum(x, n, comm);
    return hookFn ? hookFn(hookCtx, site, iter, op, x, y, n, s) : s;
}

/* normFactor: LDU/lduMatrix/lduMatrixSolver.C:183-236 */
double orc_normFactor(const orc_matrix *m, const double *psi, const double *source,
                      const double *Apsi, double *tmp, const orc_comm *comm)
{
    int n = m->a->nCells;
    orc_sumA(m, tmp);
    /* gAverage: gpuFieldCommonFunctions.C:611-635 -- global sum / global size */
    double s = site_sum(ORC_SITE_SUMPSI, 0, ORC_RED_SUM, psi, NULL, n, comm);
    double cnt = (comm && comm->nCellsGlobal) ? (double)comm->nCellsGlobal : (double)n;
    double avg = s / cnt;
    double factor = 0;
    for (int c = 0; c < n; c++) {
        double t = avg * tmp[c];
        factor += fabs(Apsi[c] - t) + fabs(source[c] - t);
    }
    if (comm && comm->sum) comm->sum(comm->ctx, &factor, 1);
    if (hookFn) {
        double *terms = (double *)malloc(sizeof(double) * (size_t)(n > 0 ? 2 * n : 1));
        for (int c = 0; c < n; c++) {
            double t = avg * tmp[c];
            terms[2 * c] = Apsi[c] - t;
            terms[2 * c + 1] = source[c] - t;
        }
        factor = hookFn(hookCtx, ORC_SITE_NORMFACTOR, 0, ORC_RED_MAG, terms, NULL, 2 * n, factor);
        free(terms);
    }
    return factor + ORC_SMALL;
}

/* ------------------------------------------------------------------------- */
/* preconditioners                                                             */
/* ------------------------------------------------------------------------- */

/* kind 0: noPreconditioner.C:58-72 ; 1: diagonalPreconditioner.C:47-89 ;
 * 2: AINVPreconditioner.C:18-117 + AINVPreconditionerF.H:42-99 */
void orc_precondition(const orc_matrix *m, int kind, int transpose, const double *rD,
                      const double *r, double *w)
{
    const orc_addr *a = m->a;
    int n = a->nCells;
    if (kind == 0) {
        for (int c = 0; c < n; c++) w[c] = r[c];
    } else if (kind == 1) {
        for (int c = 0; c < n; c++) w[c] = rD[c] * r[c];
    } else {
        const double *U = transpose ? m->lower : m->upper; /* AINVPreconditioner.C:64-72 */
        const double *L = transpose ? m->upper : m->lower;
        for (int c = 0; c < n; c++) {
            double out = 0.0;
            for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++) {
                int nb = a->u[f];
                double p = stagedAinv ? U[f] * (rD[nb] * r[nb]) : (U[f] * rD[nb]) * r[nb];
                out = out + p;
            }
            for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++) {
                int f = a->losort[k];
                int nb = a->l[f];
                double p = stagedAinv ? L[f] * (rD[nb] * r[nb]) : (L[f] * rD[nb]) * r[nb];
                out = out + p;
            }
            w[c] = rD[c] * (r[c] - out);
        }
    }
}

/* name -> kind with the reference's aliasing: lduMatrixPreconditioner.C:40-65
 * (DIC and DILU are silently replaced by AINV :58-61) */
int orc_precond_kind(const char *name, char *printed)
{
    if (!name || !*name || !strcmp(name, "none")) {
        strcpy(printed, "none");
        return 0;
    }
    if (!strcmp(name, "diagonal")) {
        strcpy(printed, "diagonal");
        return 1;
    }
    if (!strcmp(name, "AINV") || !strcmp(name, "DIC") || !strcmp(name, "DILU")) {
        strcpy(printed, "AINV");
        return 2;
    }
    return -1;
}

/* Jacobi sweep: JacobiSmoother.C:39-148, JacobiSmootherF.H:51-109 */
void orc_jacobi_smooth(const orc_matrix *m, double omega, double *psi, const double *source,
                       int nSweeps, const orc_comm *comm)
{
    const orc_addr *a = m->a;
    int n = a->nCells;
    double *Apsi = (double *)malloc(sizeof(double) * (size_t)n);
    double *b = (double *)malloc(sizeof(double) * (size_t)n);
    for (int sweep = 0; sweep < nSweeps; sweep++) {
        memcpy(b, source, sizeof(double) * (size_t)n); /* sourceTmp = source :73 */
        double *pnf = orc_halo_exchange(a, psi, comm);
        if (pnf) { /* negate = true :75-93 */
            orc_apply_interfaces(a, m->bou, pnf, b, 1);
            free(pnf);
        }
        for (int c = 0; c < n; c++) {
            double rD = 1.0 / m->diag[c];
            double t1 = (1 - omega) * psi[c];
            double t2 = (omega * rD) * b[c];
            double extra = t1 + t2;
            double out = orc_row_sum(a, c, 0.0, m->upper, m->lower, psi);
            double t3 = (omega * rD) * out;
            Apsi[c] = extra - t3;
        }
        memcpy(psi, Apsi, sizeof(double) * (size_t)n); /* psi = Apsi :146 */
    }
    free(Apsi);
    free(b);
}

/* ------------------------------------------------------------------------- */
/* solvers                                                                     */
/* ------------------------------------------------------------------------- */

/* SolverPerformance.C:74-85 */
static int orc_converged(orc_perf *p, double tol, double relTol)
{
    if (p->finalResidual < tol || (relTol > ORC_SMALL && p->finalResidual < relTol * p->initialResidual))
        p->converged = 1;
    else
        p->converged = 0;
    return p->converged;
}

/* SolverPerformance.C:32-43 */
static int orc_singular(orc_perf *p, double v)
{
    p->singular = (v < ORC_VSMALL);
    return p->singular;
}

static void hist_put(double *hist, int cap, int i, double v)
{
    if (hist && i < cap) hist[i] = v;
}

static double *vnew(int n) { return (double *)calloc((size_t)(n > 0 ? n : 1), sizeof(double)); }

static double *make_rD(const orc_matrix *m)
{
    int n = m->a->nCells;
    double *rD = vnew(n);
    for (int c = 0; c < n; c++) rD[c] = 1.0 / m->diag[c]; /* AINVPreconditioner.C:34-41 */
    return rD;
}

/* PCG: LDU/solvers/PCG/PCG.C:69-208 */
static int orc_pcg(const orc_matrix *m, int pk, const orc_controls *c, double *psi,
                   const double *source, const orc_comm *comm, orc_perf *perf, double *hist,
                   int cap)
{
    int n = m->a->nCells;
    double *pA = vnew(n), *wA = vnew(n), *rA = vnew(n);
    double wArA = ORC_GREAT, wArAold = wArA;

    orc_amul(m, psi, wA, comm);
    for (int i = 0; i < n; i++) rA[i] = source[i] - wA[i];
    double normFactor = orc_normFactor(m, psi, source, wA, pA, comm);
    perf->normFactor = normFactor;
    perf->initialResidual = site_sum(ORC_SITE_SUMMAG0, 0, ORC_RED_MAG, rA, NULL, n, comm) / normFactor;
    perf->finalResidual = perf->initialResidual;
    hist_put(hist, cap, 0, perf->finalResidual);

    if (c->minIter > 0 || !orc_converged(perf, c->tolerance, c->relTol)) {
        double *rD = make_rD(m);
        do {
            const int it = perf->nIterations;
            wArAold = wArA;
            orc_precondition(m, pk, 0, rD, rA, wA);
            wArA = site_sum(ORC_SITE_WARA, it, ORC_RED_PROD, wA, rA, n, comm);
            if (perf->nIterations == 0) {
                memcpy(pA, wA, sizeof(double) * (size_t)n);
            } else {
                double beta = wArA / wArAold;
                for (int i = 0; i < n; i++) pA[i] = fma(beta, pA[i], wA[i]);
            }
            orc_amul(m, pA, wA, comm);
            double wApA = site_sum(ORC_SITE_WAPA, it, ORC_RED_PROD, wA, pA, n, comm);
            if (orc_singular(perf, fabs(wApA) / normFactor)) break;
            double alpha = wArA / wApA;
            for (int i = 0; i < n; i++) psi[i] = fma(alpha, pA[i], psi[i]);
            for (int i = 0; i < n; i++) rA[i] = fma(-alpha, wA[i], rA[i]);
            perf->finalResidual = site_sum(ORC_SITE_SUMMAG, it, ORC_RED_MAG, rA, NULL, n, comm) / normFactor;
            hist_put(hist, cap, perf->nIterations + 1, perf->finalResidual);
        } while ((perf->nIterations++ < c->maxIter &&
                  !orc_converged(perf, c->tolerance, c->relTol)) ||
                 perf->nIterations < c->minIter);
        free(rD);
    }
    free(pA);
    free(wA);
    free(rA);
    return 0;
}

/* PBiCG: LDU/solvers/PBiCG/PBiCG.C:68-246 */
static int orc_pbicg(const orc_matrix *m, int pk, const orc_controls *c, double *psi,
                     const double *source, const orc_comm *comm, orc_perf *perf, double *hist,
                     int cap)
{
    int n = m->a->nCells;
    double *pA = vnew(n), *pT = vnew(n), *wA = vnew(n), *wT = vnew(n), *rA = vnew(n),
           *rT = vnew(n);
    double wArT = ORC_GREAT, wArTold = wArT;

    orc_amul(m, psi, wA, comm);
    orc_tmul(m, psi, wT, comm);
    for (int i = 0; i < n; i++) rA[i] = source[i] - wA[i];
    for (int i = 0; i < n; i++) rT[i] = source[i] - wT[i];
    double normFactor = orc_normFactor(m, psi, source, wA, pA, comm);
    perf->normFactor = normFactor;
    perf->initialResidual = site_sum(ORC_SITE_SUMMAG0, 0, ORC_RED_MAG, rA, NULL, n, comm) / normFactor;
    perf->finalResidual = perf->initialResidual;
    hist_put(hist, cap, 0, perf->finalResidual);

    if (c->minIter > 0 || !orc_converged(perf, c->tolerance, c->relTol)) {
        double *rD = make_rD(m);
        do {
            const int it = perf->nIterations;
            wArTold = wArT;
            orc_precondition(m, pk, 0, rD, rA, wA);
            orc_precondition(m, pk, 1, rD, rT, wT);
            wArT = site_sum(ORC_SITE_WART, it, ORC_RED_PROD, wA, rT, n, comm);
            if (perf->nIterations == 0) {
                memcpy(pA, wA, sizeof(double) * (size_t)n);
                memcpy(pT, wT, sizeof(double) * (size_t)n);
            } else {
                double beta = wArT / wArTold;
                for (int i = 0; i < n; i++) pA[i] = fma(beta, pA[i], wA[i]);
                for (int i = 0; i < n; i++) pT[i] = fma(beta, pT[i], wT[i]);
            }
            orc_amul(m, pA, wA, comm);
            orc_tmul(m, pT, wT, comm);
            double wApT = site_sum(ORC_SITE_WAPT, it, ORC_RED_PROD, wA, pT, n, comm);
            if (orc_singular(perf, fabs(wApT) / normFactor)) break;
            double alpha = wArT / wApT;
            for (int i = 0; i < n; i++) psi[i] = fma(alpha, pA[i], psi[i]);
            for (int i = 0; i < n; i++) rA[i] = fma(-alpha, wA[i], rA[i]);
            for (int i = 0; i < n; i++) rT[i] = fma(-alpha, wT[i], rT[i]);
            perf->finalResidual = site_sum(ORC_SITE_SUMMAG, it, ORC_RED_MAG, rA, NULL, n, comm) / normFactor;
            hist_put(hist, cap, perf->nIterations + 1, perf->finalResidual);
        } while ((perf->nIterations++ < c->maxIter &&
                  !orc_converged(perf, c->tolerance, c->relTol)) ||
                 perf->nIterations < c->minIter);
        free(rD);
    }
    free(pA);
    free(pT);
    free(wA);
    free(wT);
    free(rA);
    free(rT);
    return 0;
}

/* PBiCGStab: LDU/solvers/PBiCGStab/PBiCGStab.C:66-300.  The reference's second
 * solution update passes yA where zA is meant (:263-270); bicgstabRefQuirk = 1
 * mirrors that, 0 (default) uses zA. */
static int orc_pbicgstab(const orc_matrix *m, int pk, const orc_controls *c, double *psi,
                         const double *source, const orc_comm *comm, orc_perf *perf,
                         double *hist, int cap)
{
    int n = m->a->nCells;
    double *pA = vnew(n), *yA = vnew(n), *rA = vnew(n);
    orc_amul(m, psi, yA, comm);
    for (int i = 0; i < n; i++) rA[i] = source[i] - yA[i];
    double normFactor = orc_normFactor(m, psi, source, yA, pA, comm);
    perf->normFactor = normFactor;
    perf->initialResidual = site_sum(ORC_SITE_SUMMAG0, 0, ORC_RED_MAG, rA, NULL, n, comm) / normFactor;
    perf->finalResidual = perf->initialResidual;
    hist_put(hist, cap, 0, perf->finalResidual);

    if (c->minIter > 0 || !orc_converged(perf, c->tolerance, c->relTol)) {
        double *AyA = vnew(n), *sA = vnew(n), *zA = vnew(n), *tA = vnew(n), *rA0 = vnew(n);
        double *rD = make_rD(m);
        memcpy(rA0, rA, sizeof(double) * (size_t)n);
        double rA0rA = 0, alpha = 0, omega = 0;
        int early = 0;
        do {
            const int it = perf->nIterations;
            double rA0rAold = rA0rA;
            rA0rA = site_sum(ORC_SITE_RA0RA, it, ORC_RED_PROD, rA0, rA, n, comm);
            if (orc_singular(perf, fabs(rA0rA))) break;
            if (perf->nIterations == 0) {
                memcpy(pA, rA, sizeof(double) * (size_t)n);
            } else {
                if (orc_singular(perf, fabs(omega))) break;
                double beta = (rA0rA / rA0rAold) * (alpha / omega);
                for (int i = 0; i < n; i++) {
                    double r1 = fma(-omega, AyA[i], pA[i]); /* result1 = pA - omega*AyA */
                    pA[i] = fma(beta, r1, rA[i]);
                }
            }
            orc_precondition(m, pk, 0, rD, pA, yA);
            orc_amul(m, yA, AyA, comm);
            double rA0AyA = site_sum(ORC_SITE_RA0AYA, it, ORC_RED_PROD, rA0, AyA, n, comm);
            alpha = rA0rA / rA0AyA;
            for (int i = 0; i < n; i++) sA[i] = fma(-alpha, AyA[i], rA[i]);
            perf->finalResidual = site_sum(ORC_SITE_SUMMAGS, it, ORC_RED_MAG, sA, NULL, n, comm) / normFactor;
            if (orc_converged(perf, c->tolerance, c->relTol)) {
                for (int i = 0; i < n; i++) psi[i] = fma(alpha, yA[i], psi[i]);
                perf->nIterations++;
                hist_put(hist, cap, perf->nIterations, perf->finalResidual);
                early = 1;
                break;
            }
            orc_precondition(m, pk, 0, rD, sA, zA);
            orc_amul(m, zA, tA, comm);
            double tAtA = site_sum(ORC_SITE_TATA, it, ORC_RED_PROD, tA, tA, n, comm);
            omega = site_sum(ORC_SITE_TASA, it, ORC_RED_PROD, tA, sA, n, comm) / tAtA;
            for (int i = 0; i < n; i++) psi[i] = fma(alpha, yA[i], psi[i]);
            {
                const double *second = c->bicgstabRefQuirk ? yA : zA;
                for (int i = 0; i < n; i++) psi[i] = fma(omega, second[i], psi[i]);
            }
            for (int i = 0; i < n; i++) rA[i] = fma(-omega, tA[i], sA[i]);
            perf->finalResidual = site_sum(ORC_SITE_SUMMAG, it, ORC_RED_MAG, rA, NULL, n, comm) / normFactor;
            hist_put(hist, cap, perf->nIterations + 1, perf->finalResidual);
        } while ((perf->nIterations++ < c->maxIter &&
                  !orc_converged(perf, c->tolerance, c->relTol)) ||
                 perf->nIterations < c->minIter);
        (void)early;
        free(AyA);
        free(sA);
        free(zA);
        free(tA);
        free(rA0);
        free(rD);
    }
    free(pA);
    free(yA);
    free(rA);
    return 0;
}

/* smoothSolver: LDU/solvers/smoothSolver/smoothSolver.C:77-193 (smoother Jacobi;
 * "GaussSeidel" aliases to it, GaussSeidelSmoother.C:43-69) */
static int orc_smooth_solver(const orc_matrix *m, const orc_controls *c, double *psi,
                             const double *source, const orc_comm *comm, orc_perf *perf,
                             double *hist, int cap)
{
    int n = m->a->nCells;
    if (c->nSweeps < 0) {
        orc_jacobi_smooth(m, c->omega, psi, source, -c->nSweeps, comm);
        perf->nIterations -= c->nSweeps;
        return 0;
    }
    double *Apsi = vnew(n), *tmp = vnew(n);
    orc_amul(m, psi, Apsi, comm);
    double normFactor = orc_normFactor(m, psi, source, Apsi, tmp, comm);
    perf->normFactor = normFactor;
    for (int i = 0; i < n; i++) tmp[i] = source[i] - Apsi[i];
    perf->initialResidual = site_sum(ORC_SITE_SUMMAG0, 0, ORC_RED_MAG, tmp, NULL, n, comm) / normFactor;
    perf->finalResidual = perf->initialResidual;
    hist_put(hist, cap, 0, perf->finalResidual);
    if (c->minIter > 0 || !orc_converged(perf, c->tolerance, c->relTol)) {
        int k = 0;
        do {
            orc_jacobi_smooth(m, c->omega, psi, source, c->nSweeps, comm);
            orc_residual(m, psi, source, tmp, comm);
            perf->finalResidual = site_sum(ORC_SITE_SUMMAG, k, ORC_RED_MAG, tmp, NULL, n, comm) / normFactor;
            hist_put(hist, cap, ++k, perf->finalResidual);
        } while (((perf->nIterations += c->nSweeps) < c->maxIter &&
                  !orc_converged(perf, c->tolerance, c->relTol)) ||
                 perf->nIterations < c->minIter);
    }
    free(Apsi);
    free(tmp);
    return 0;
}

/* run-time selection: LDU/lduMatrix/lduMatrixSolver.C:43-140.  Returns 0 on success,
 * -1 unknown solver, -2 unknown preconditioner/smoother, -3 wrong matrix kind. */
int orc_solve(const orc_matrix *m, const char *solver, const char *pre, const orc_controls *c,
              double *psi, const double *source, const orc_comm *comm, orc_perf *perf,
              double *hist, int histCap)
{
    memset(perf, 0, sizeof(*perf));
    int n = m->a->nCells;
    char pname[32];
    int diagonalOnly = (m->a->nFaces == 0);
    if (diagonalOnly || !strcmp(solver, "diagonal")) { /* diagonalSolver.C:62-81 */
        for (int i = 0; i < n; i++) psi[i] = source[i] / m->diag[i];
        strcpy(perf->solverName, "diagonal");
        perf->converged = 1;
        return 0;
    }
    /* ICCG / BICCG wrappers: ICCG.C:40-51 = PCG + DIC, BICCG = PBiCG + DILU */
    if (!strcmp(solver, "ICCG")) {
        solver = "PCG";
        pre = "DIC";
    } else if (!strcmp(solver, "BICCG")) {
        solver = "PBiCG";
        pre = "DILU";
    }
    if (!strcmp(solver, "PCG") || !strcmp(solver, "PBiCG") || !strcmp(solver, "PBiCGStab")) {
        /* solver::New looks the name up in the table of the matrix kind first (lduMatrixSolver.C:70-133):
         * PCG symmetric only (PCG.C:36), PBiCG / PBiCGStab asymmetric only (PBiCG.C:36, PBiCGStab.C:36) */
        int wantSym = !strcmp(solver, "PCG");
        if (wantSym != (m->symmetric ? 1 : 0)) return -3;
        /* preconditioner::New inside solve(): DIC is registered for symmetric matrices, DILU for asymmetric
         * ones, AINV / diagonal / none for both (DICPreconditioner.C:35, DILUPreconditioner.C:35, ...) */
        int pk = orc_precond_kind(pre, pname);
        if (pk < 0) return -2;
        if (pre && ((!strcmp(pre, "DILU") && m->symmetric) || (!strcmp(pre, "DIC") && !m->symmetric))) return -2;
        snprintf(perf->solverName, sizeof(perf->solverName), "%s%s", pname, solver);
        if (!strcmp(solver, "PCG")) return orc_pcg(m, pk, c, psi, source, comm, perf, hist, histCap);
        if (!strcmp(solver, "PBiCG")) return orc_pbicg(m, pk, c, psi, source, comm, perf, hist, histCap);
        return orc_pbicgstab(m, pk, c, psi, source, comm, perf, hist, histCap);
    }
    if (!strcmp(solver, "smoothSolver")) {
        if (pre && *pre && strcmp(pre, "Jacobi") && strcmp(pre, "GaussSeidel")) return -2;
        strcpy(perf->solverName, "smoothSolver");
        return orc_smooth_solver(m, c, psi, source, comm, perf, hist, histCap);
    }
    return -1;
}

/* accessors for tests */
const int *orc_addr_lower(const orc_addr *a) { return a->l; }
const int *orc_addr_upper(const orc_addr *a) { return a->u; }
int orc_addr_npatches(const orc_addr *a) { return a->nPatches; }
const int *orc_addr_patch_start(const orc_addr *a) { return a->patchStart; }
const int *orc_addr_face_cells(const orc_addr *a) { return a->faceCells; }
