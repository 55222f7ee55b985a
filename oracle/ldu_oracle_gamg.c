/*
 * ldu_oracle_gamg.c -- CPU restatement of the RapidCFD-dev GAMG solver (pair
 * agglomeration, coarse addressing, Galerkin-by-summation coarse matrices, V-cycle).
 * TEST INFRASTRUCTURE ONLY (see ldu_oracle.h: V-cycle, pair agglomeration, coarse addressing,
 * combineLevels, coarse matrices, coarse processor interfaces and the LU are pinned to the
 * reference's own code, tests/test_reference_functors.py).
 *
 * Paths relative to /root/reference/src/OpenFOAM/matrices/lduMatrix/solvers/GAMG/
 * (abbreviated GAMG/).  Multi-rank: processor interfaces are agglomerated as in
 * interfaces/processorGAMGInterface/processorGAMGInterface.C:60-140 (unique (master cell,
 * slave cell) pairs in order of first appearance along the fine patch), their coefficients
 * are restricted by summation (GAMGSolverAgglomerateMatrix.C:325-447) and the coarsest
 * level is solved directly on the matrix assembled from all ranks (LUscalarMatrix.C:60-160;
 * here every rank assembles and factorises the same global matrix instead of the master).
 */
#include "ldu_oracle_internal.h"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define ORC_MAX_LEVELS 50 /* GAMGAgglomeration.C:94 maxLevels_(50) */

struct orc_gamg {
    int nLevels;                       /* coarse levels created */
    orc_addr *addr[ORC_MAX_LEVELS];    /* coarse level addressing, [0] = first coarse */
    int *restrictAddr[ORC_MAX_LEVELS]; /* cells of level k (0 = finest) -> cells of coarse k */
    int *faceRestrict[ORC_MAX_LEVELS]; /* faces of level k -> coarse face or -(cell+1) */
    unsigned char *faceFlip[ORC_MAX_LEVELS];
    int nFineCells[ORC_MAX_LEVELS], nFineFaces[ORC_MAX_LEVELS];
    int *patchFaceRestrict[ORC_MAX_LEVELS]; /* fine patch face (flat) -> coarse patch face (flat) */
    int nFinePatchFaces[ORC_MAX_LEVELS];
    const orc_addr *finest;
    /* opt-in coarsest solve with a given inverse (orc_gamg_set_coarsest_inverse) */
    double *devInv; /* this rank's rows of the inverse, row-major nCoarsest x devN */
    int *devPerm;   /* banded row of every coarsest cell */
    int devN;
    int scaleDescending; /* orc_gamg_set_scale_order */
};

/* pairGAMGAgglomeration::agglomerate(nCoarseCells, addr, faceWeights):
 * GAMGAgglomerations/pairGAMGAgglomeration/pairGAMGAgglomerate.C:135-313 */
static int *pair_agglomerate(const orc_addr *a, const double *w, int *nCoarseOut, int *forward)
{
    int n = a->nCells, nf = a->nFaces;
    const int *up = a->u, *lo = a->l;
    int *off = (int *)calloc((size_t)n + 1, sizeof(int));
    int *cnt = (int *)calloc((size_t)n + 1, sizeof(int));
    int *cf = (int *)malloc(sizeof(int) * (size_t)(2 * nf + 1));
    for (int f = 0; f < nf; f++) cnt[up[f]]++;
    for (int f = 0; f < nf; f++) cnt[lo[f]]++;
    for (int c = 0; c < n; c++) off[c + 1] = off[c] + cnt[c];
    memset(cnt, 0, sizeof(int) * ((size_t)n + 1));
    /* per cell: first the faces where it is neighbour (upperAddr hits), then the
     * faces it owns (:172-192) */
    for (int f = 0; f < nf; f++) cf[off[up[f]] + cnt[up[f]]++] = f;
    for (int f = 0; f < nf; f++) cf[off[lo[f]] + cnt[lo[f]]++] = f;

    int *map = (int *)malloc(sizeof(int) * (size_t)(n > 0 ? n : 1));
    for (int c = 0; c < n; c++) map[c] = -1;
    int nCoarse = 0;
    const double GREAT = 1e20;
    for (int ci = 0; ci < n; ci++) {
        int c = *forward ? ci : n - ci - 1;
        if (map[c] >= 0) continue;
        int match = -1;
        double maxW = -GREAT;
        for (int k = off[c]; k < off[c + 1]; k++) {
            int f = cf[k];
            if (map[up[f]] < 0 && map[lo[f]] < 0 && w[f] > maxW) {
                match = f;
                maxW = w[f];
            }
        }
        if (match >= 0) {
            map[up[match]] = nCoarse;
            map[lo[match]] = nCoarse;
            nCoarse++;
        } else {
            int cm = -1;
            double cmax = -GREAT;
            for (int k = off[c]; k < off[c + 1]; k++) {
                int f = cf[k];
                if (w[f] > cmax) {
                    cm = f;
                    cmax = w[f];
                }
            }
            if (cm >= 0) {
                int a1 = map[up[cm]], a2 = map[lo[cm]];
                map[c] = a1 > a2 ? a1 : a2;
            }
        }
    }
    for (int ci = 0; ci < n; ci++) { /* leftover singletons :276-286 */
        int c = *forward ? ci : n - ci - 1;
        if (map[c] < 0) map[c] = nCoarse++;
    }
    if (!*forward) { /* :288-298 */
        nCoarse--;
        for (int c = 0; c < n; c++) map[c] = nCoarse - map[c];
        nCoarse++;
    }
    *forward = !*forward; /* :302-304 static direction flag */
    free(off);
    free(cnt);
    free(cf);
    *nCoarseOut = nCoarse;
    return map;
}

/* GAMGAgglomeration::agglomerateLduAddressing:
 * GAMGAgglomerations/GAMGAgglomeration/GAMGAgglomerateLduAddressing.C:245-461 */
static orc_addr *coarse_addressing(const orc_addr *fine, const int *rmap, int nCoarse,
                                   int **faceRestrictOut, unsigned char **flipOut)
{
    int nff = fine->nFaces;
    int maxN = 10;
    int *ccn = (int *)calloc((size_t)nCoarse, sizeof(int));
    int *ccf = (int *)malloc(sizeof(int) * (size_t)maxN * (size_t)nCoarse);
    int *fr = (int *)malloc(sizeof(int) * (size_t)(nff > 0 ? nff : 1));
    int *initNei = (int *)malloc(sizeof(int) * (size_t)(nff > 0 ? nff : 1));
    int nCF = 0;
    for (int f = 0; f < nff; f++) {
        int ru = rmap[fine->u[f]], rl = rmap[fine->l[f]];
        if (ru == rl) {
            fr[f] = -(ru + 1);
            continue;
        }
        int cOwn = ru, cNei = rl;
        if (ru > rl) {
            cOwn = rl;
            cNei = ru;
        }
        int found = 0;
        for (int i = 0; i < ccn[cOwn]; i++) {
            int cfi = ccf[(size_t)maxN * cOwn + i];
            if (initNei[cfi] == cNei) {
                found = 1;
                fr[f] = cfi;
                break;
            }
        }
        if (!found) {
            if (ccn[cOwn] >= maxN) {
                int oldN = maxN;
                maxN *= 2;
                ccf = (int *)realloc(ccf, sizeof(int) * (size_t)maxN * (size_t)nCoarse);
                for (int i = nCoarse - 1; i >= 0; i--)
                    for (int j = ccn[i] - 1; j >= 0; j--)
                        ccf[(size_t)maxN * i + j] = ccf[(size_t)oldN * i + j];
            }
            ccf[(size_t)maxN * cOwn + ccn[cOwn]] = nCF;
            initNei[nCF] = cNei;
            fr[f] = nCF;
            ccn[cOwn]++;
            nCF++;
        }
    }
    /* renumber grouped by coarse owner, discovery order within an owner (:381-402) */
    int *cOwner = (int *)malloc(sizeof(int) * (size_t)(nCF > 0 ? nCF : 1));
    int *cNeigh = (int *)malloc(sizeof(int) * (size_t)(nCF > 0 ? nCF : 1));
    int *cMap = (int *)malloc(sizeof(int) * (size_t)(nCF > 0 ? nCF : 1));
    int k = 0;
    for (int cc = 0; cc < nCoarse; cc++)
        for (int i = 0; i < ccn[cc]; i++) {
            int cfi = ccf[(size_t)maxN * cc + i];
            cOwner[k] = cc;
            cNeigh[k] = initNei[cfi];
            cMap[cfi] = k;
            k++;
        }
    for (int f = 0; f < nff; f++)
        if (fr[f] >= 0) fr[f] = cMap[fr[f]];
    unsigned char *flip = (unsigned char *)calloc((size_t)(nff > 0 ? nff : 1), 1);
    for (int f = 0; f < nff; f++) { /* :413-446 */
        if (fr[f] >= 0) {
            int ru = rmap[fine->u[f]], rl = rmap[fine->l[f]];
            if (cOwner[fr[f]] == ru && cNeigh[fr[f]] == rl) flip[f] = 1;
        }
    }
    orc_addr *ca = orc_addr_create(nCoarse, nCF, cOwner, cNeigh, 0, NULL, NULL);
    free(ccn);
    free(ccf);
    free(initNei);
    free(cOwner);
    free(cNeigh);
    free(cMap);
    *faceRestrictOut = fr;
    *flipOut = flip;
    return ca;
}

/* processorGAMGInterface / cyclicGAMGInterface: coarse patch faces of every coupled patch
 * (interfaces/processorGAMGInterface/processorGAMGInterface.C:60-140, cyclicGAMGInterface/cyclicGAMGInterface.C:70-150).  nbrMap holds the
 * neighbour side's restrict-map values per fine patch face (internalFieldTransfer). */
static void coarse_interfaces(const orc_addr *fine, const int *rmap, const double *nbrMap, int myRank,
                              int **cPatchStartOut, int **cFaceCellsOut, int **pfRestrictOut)
{
    int nP = fine->nPatches;
    int tot = nP ? fine->patchStart[nP] : 0;
    int *cStart = (int *)calloc((size_t)nP + 1, sizeof(int));
    int *cCells = (int *)malloc(sizeof(int) * (size_t)(tot > 0 ? tot : 1));
    int *pfr = (int *)malloc(sizeof(int) * (size_t)(tot > 0 ? tot : 1));
    int nC = 0;
    for (int p = 0; p < nP; p++) {
        int s0 = fine->patchStart[p], s1 = fine->patchStart[p + 1];
        int nb = fine->neighbRank ? fine->neighbRank[p] : -1;
        cStart[p] = nC;
        /* pairs (master cell, slave cell); linear search keeps first-appearance order */
        int *pa = (int *)malloc(sizeof(int) * (size_t)(s1 - s0 + 1));
        int *pb = (int *)malloc(sizeof(int) * (size_t)(s1 - s0 + 1));
        int np = 0;
        for (int i = s0; i < s1; i++) {
            int mine = rmap[fine->faceCells[i]], theirs = (int)nbrMap[i];
            /* master side first so that both sides enumerate the same pairs: the lower rank for a processor patch
             * (processorGAMGInterface.C:93-118), the owner patch = lower patch index for a cyclic pair
             * (cyclicGAMGInterface.C:104-127; nb = -(q+1), cyclicLduInterface::owner()) */
            int master = nb >= 0 ? (myRank < nb) : (p < -nb - 1);
            int a = master ? mine : theirs, b = master ? theirs : mine;
            int found = -1;
            for (int k = np - 1; k >= 0; k--) /* recent pairs first: patches are locally ordered */
                if (pa[k] == a && pb[k] == b) {
                    found = k;
                    break;
                }
            if (found < 0) {
                found = np;
                pa[np] = a;
                pb[np] = b;
                cCells[nC + np] = mine;
                np++;
            }
            pfr[i] = nC + found;
        }
        nC += np;
        free(pa);
        free(pb);
    }
    cStart[nP] = nC;
    *cPatchStartOut = cStart;
    *cFaceCellsOut = cCells;
    *pfRestrictOut = pfr;
}

/* level loop: pairGAMGAgglomerate.C:31-130 (mergeLevels 1 only) */
/* combineLevels: GAMGAgglomerateLduAddressing.C:606-765.  Level cur (built on the coarse
 * addressing of level cur-1) is folded into level cur-1: cell, face and patch-face maps are
 * composed and the coarser addressing replaces the intermediate one.  As in the reference the
 * flip of a composed face is the flip of the SECOND step alone (:631), not the exclusive-or of
 * the two; the flip of a face that collapses into a cell is never read (the reference indexes
 * the face flip list with a cell label there, :637) and is stored as 0. */
static void combine_levels(orc_gamg *g, int cur)
{
    int prev = cur - 1;
    int *pr = g->restrictAddr[prev], *cr = g->restrictAddr[cur];
    int *pf = g->faceRestrict[prev], *cf = g->faceRestrict[cur];
    unsigned char *pflip = g->faceFlip[prev], *cflip = g->faceFlip[cur];
    for (int i = 0; i < g->nFineFaces[prev]; i++) {
        if (pf[i] >= 0) {
            int mid = pf[i];
            pf[i] = cf[mid];
            pflip[i] = cflip[mid];
        } else {
            int midCell = -pf[i] - 1;
            pf[i] = -cr[midCell] - 1;
            pflip[i] = 0;
        }
    }
    for (int i = 0; i < g->nFineCells[prev]; i++) pr[i] = cr[pr[i]];
    if (g->patchFaceRestrict[prev] && g->patchFaceRestrict[cur])
        for (int i = 0; i < g->nFinePatchFaces[prev]; i++)
            g->patchFaceRestrict[prev][i] = g->patchFaceRestrict[cur][g->patchFaceRestrict[prev][i]];
    orc_addr_free(g->addr[prev]);
    g->addr[prev] = g->addr[cur];
    g->addr[cur] = NULL;
    free(cr);
    free(cf);
    free(cflip);
    free(g->patchFaceRestrict[cur]);
    g->restrictAddr[cur] = NULL;
    g->faceRestrict[cur] = NULL;
    g->faceFlip[cur] = NULL;
    g->patchFaceRestrict[cur] = NULL;
}

orc_gamg *orc_gamg_create(const orc_addr *a, const double *faceWeights,
                          int nCellsInCoarsestLevel, int mergeLevels, int *forwardFlag,
                          const orc_comm *comm)
{
    if (mergeLevels < 1) return NULL;
    int nPairLevels = 0;
    orc_gamg *g = (orc_gamg *)calloc(1, sizeof(orc_gamg));
    g->finest = a;
    int fwd_local = 1; /* pairGAMGAgglomeration.C:33 initial forward_ = true */
    int *fwd = forwardFlag ? forwardFlag : &fwd_local;
    const orc_addr *fine = a;
    double *w = (double *)malloc(sizeof(double) * (size_t)(a->nFaces > 0 ? a->nFaces : 1));
    memcpy(w, faceWeights, sizeof(double) * (size_t)a->nFaces);
    while (g->nLevels < ORC_MAX_LEVELS - 1) {
        int nCoarse = -1;
        int *map = pair_agglomerate(fine, w, &nCoarse, fwd);
        /* continueAgglomerating: GAMGAgglomeration.C:72-84 (and-reduced over the ranks) */
        double stopVotes = (nCoarse >= nCellsInCoarsestLevel) ? 0.0 : 1.0;
        if (comm && comm->sum) comm->sum(comm->ctx, &stopVotes, 1);
        if (stopVotes > 0) {
            free(map);
            break;
        }
        int lev = g->nLevels;
        g->restrictAddr[lev] = map;
        g->nFineCells[lev] = fine->nCells;
        g->nFineFaces[lev] = fine->nFaces;
        g->addr[lev] = coarse_addressing(fine, map, nCoarse, &g->faceRestrict[lev], &g->faceFlip[lev]);
        g->nFinePatchFaces[lev] = fine->nPatches ? fine->patchStart[fine->nPatches] : 0;
        if (fine->nPatches) { /* GAMGAgglomerateLduAddressing.C:470-560 */
            int tot = fine->patchStart[fine->nPatches];
            double *mapD = (double *)malloc(sizeof(double) * (size_t)fine->nCells);
            for (int c = 0; c < fine->nCells; c++) mapD[c] = (double)map[c];
            double *nbrMap = orc_halo_exchange(fine, mapD, comm);
            free(mapD);
            int *cStart, *cCells;
            coarse_interfaces(fine, map, nbrMap, comm ? comm->rank : 0, &cStart, &cCells,
                              &g->patchFaceRestrict[lev]);
            free(nbrMap);
            /* rebuild the coarse addressing with its coupled patches */
            orc_addr *ca = g->addr[lev];
            orc_addr *withP = orc_addr_create(ca->nCells, ca->nFaces, ca->l, ca->u, fine->nPatches, cStart, cCells);
            if (fine->neighbRank) orc_addr_set_neighb_ranks(withP, fine->neighbRank);
            orc_addr_free(ca);
            g->addr[lev] = withP;
            free(cStart);
            free(cCells);
            (void)tot;
        }
        /* restrictFaceField of the weights (:86-107; GAMGAgglomerationTemplates.C:155-271) */
        double *cw = (double *)calloc((size_t)(g->addr[lev]->nFaces > 0 ? g->addr[lev]->nFaces : 1),
                                      sizeof(double));
        for (int f = 0; f < fine->nFaces; f++)
            if (g->faceRestrict[lev][f] >= 0) cw[g->faceRestrict[lev][f]] += w[f];
        free(w);
        w = cw;
        fine = g->addr[lev];
        if (nPairLevels % mergeLevels) /* pairGAMGAgglomerate.C:110-117 */
            combine_levels(g, lev);
        else
            g->nLevels++;
        nPairLevels++;
    }
    free(w);
    return g;
}

void orc_gamg_free(orc_gamg *g)
{
    if (!g) return;
    for (int i = 0; i < g->nLevels; i++) {
        orc_addr_free(g->addr[i]);
        free(g->restrictAddr[i]);
        free(g->faceRestrict[i]);
        free(g->faceFlip[i]);
        free(g->patchFaceRestrict[i]);
    }
    free(g->devInv);
    free(g->devPerm);
    free(g);
}

int orc_gamg_nlevels(const orc_gamg *g) { return g->nLevels; }
int orc_gamg_ncells(const orc_gamg *g, int lev) { return g->addr[lev]->nCells; }
int orc_gamg_nfaces(const orc_gamg *g, int lev) { return g->addr[lev]->nFaces; }
int orc_gamg_npatchfaces(const orc_gamg *g, int lev)
{
    const orc_addr *a = g->addr[lev];
    return a->nPatches ? a->patchStart[a->nPatches] : 0;
}
const int *orc_gamg_restrict_addr(const orc_gamg *g, int lev) { return g->restrictAddr[lev]; }
const int *orc_gamg_face_restrict_addr(const orc_gamg *g, int lev) { return g->faceRestrict[lev]; }
const unsigned char *orc_gamg_face_flip(const orc_gamg *g, int lev) { return g->faceFlip[lev]; }
const orc_addr *orc_gamg_addr(const orc_gamg *g, int lev) { return g->addr[lev]; }
const int *orc_gamg_patch_face_restrict(const orc_gamg *g, int lev) { return g->patchFaceRestrict[lev]; }

/* GAMGInterface::agglomerateCoeffs (GAMGInterface.C:120-172; segments of a stable sort: ascending fine index) */
void orc_gamg_agglomerate_patch_coeffs(const orc_gamg *g, int lev, const double *fine, double *coarse)
{
    const orc_addr *ca = g->addr[lev];
    int nCP = ca->nPatches ? ca->patchStart[ca->nPatches] : 0;
    for (int i = 0; i < nCP; i++) coarse[i] = 0.0;
    for (int i = 0; i < g->nFinePatchFaces[lev]; i++) {
        int cpf = g->patchFaceRestrict[lev][i];
        coarse[cpf] = coarse[cpf] + fine[i];
    }
}

/* restrictField: GAMGAgglomerationTemplates.C:35-61, GAMGAgglomerationF.H:10-40.
 * Segments come from a stable sort, so each coarse value is the sum of its fine
 * values in ascending fine index starting from zero. */
static void restrict_field(const int *map, int nFine, int nCoarse, const double *ff, double *cf)
{
    for (int i = 0; i < nCoarse; i++) cf[i] = 0.0;
    for (int i = 0; i < nFine; i++) cf[map[i]] = cf[map[i]] + ff[i];
}

/* prolongField: GAMGAgglomerationTemplates.C:273-308 */
static void prolong_field(const int *map, int nFine, const double *cf, double *ff)
{
    for (int i = 0; i < nFine; i++) ff[i] = cf[map[i]];
}

typedef struct {
    int n, nf;
    double *diag, *upper, *lower; /* lower == NULL when symmetric */
    double *bou, *intc;           /* coupled-patch coefficients of this level */
    orc_matrix *m;
} lev_matrix;

/* agglomerateMatrix: GAMGSolverAgglomerateMatrix.C:37-322 with the sorted
 * (non-atomic) functors GAMGSolverAgglomerateMatrixF.H:9-160 */
static void agglomerate_matrix(const orc_gamg *g, int lev, const double *fd, const double *fu,
                               const double *fl, const double *fbou, const double *fint, lev_matrix *cm)
{
    const orc_addr *ca = g->addr[lev];
    int nFine = g->nFineCells[lev], nFF = g->nFineFaces[lev];
    cm->n = ca->nCells;
    cm->nf = ca->nFaces;
    cm->diag = (double *)calloc((size_t)cm->n, sizeof(double));
    cm->upper = (double *)calloc((size_t)(cm->nf > 0 ? cm->nf : 1), sizeof(double));
    cm->lower = fl ? (double *)calloc((size_t)(cm->nf > 0 ? cm->nf : 1), sizeof(double)) : NULL;
    restrict_field(g->restrictAddr[lev], nFine, cm->n, fd, cm->diag); /* :59-71 */
    const int *fr = g->faceRestrict[lev];
    const unsigned char *flip = g->faceFlip[lev];
    for (int f = 0; f < nFF; f++) {
        if (fr[f] >= 0) {
            if (!fl) {
                cm->upper[fr[f]] = cm->upper[fr[f]] + fu[f];
            } else if (!flip[f]) {
                cm->upper[fr[f]] = cm->upper[fr[f]] + fu[f];
                cm->lower[fr[f]] = cm->lower[fr[f]] + fl[f];
            } else {
                cm->upper[fr[f]] = cm->upper[fr[f]] + fl[f];
                cm->lower[fr[f]] = cm->lower[fr[f]] + fu[f];
            }
        } else {
            int c = -1 - fr[f];
            if (!fl)
                cm->diag[c] = cm->diag[c] + 2 * fu[f];
            else
                cm->diag[c] = cm->diag[c] + (fu[f] + fl[f]);
        }
    }
    /* agglomerateInterfaceCoefficients (:325-447): sums over the patch face map */
    int nCP = ca->nPatches ? ca->patchStart[ca->nPatches] : 0;
    cm->bou = (double *)calloc((size_t)(nCP > 0 ? nCP : 1), sizeof(double));
    cm->intc = (double *)calloc((size_t)(nCP > 0 ? nCP : 1), sizeof(double));
    if (g->nFinePatchFaces[lev] > 0) {
        orc_gamg_agglomerate_patch_coeffs(g, lev, fbou, cm->bou);
        orc_gamg_agglomerate_patch_coeffs(g, lev, fint, cm->intc);
    }
    cm->m = orc_matrix_create(ca, cm->diag, cm->upper, cm->lower, nCP ? cm->bou : NULL, nCP ? cm->intc : NULL);
}

/* scale: GAMGSolverScale.C:59-171 */
static void gamg_scale(const orc_matrix *A, double *field, double *Acf, const double *source,
                       const orc_comm *comm, int descending)
{
    int n = A->a->nCells;
    orc_amul(A, field, Acf, comm);
    double num = 0, den = 0;
    if (descending) { /* the same two sums in the other order: a measure of what any other order may change */
        for (int i = n - 1; i >= 0; i--) num += source[i] * field[i];
        for (int i = n - 1; i >= 0; i--) den += Acf[i] * field[i];
    } else {
        for (int i = 0; i < n; i++) num += source[i] * field[i];
        for (int i = 0; i < n; i++) den += Acf[i] * field[i];
    }
    if (comm && comm->sum) { /* vector2D all-reduce: GAMGSolverScale.C:139-140 */
        double v[2] = {num, den};
        comm->sum(comm->ctx, v, 2);
        num = v[0];
        den = v[1];
    }
    /* stabilise(y, VSMALL): y >= 0 ? y + VSMALL : y - VSMALL */
    double sden = den >= 0 ? den + 1e-300 : den - 1e-300;
    double sf = num / sden;
    for (int i = 0; i < n; i++) {
        double t1 = sf * field[i];
        double t2 = sf * Acf[i];
        field[i] = t1 + (source[i] - t2) / A->diag[i];
    }
}

/* interpolate (first overload): GAMGSolverInterpolate.C:45-110 */
static void gamg_interpolate(const orc_matrix *A, double *psi, double *Apsi, const orc_comm *comm)
{
    const orc_addr *a = A->a;
    double *pnf = orc_halo_exchange(a, psi, comm);
    for (int c = 0; c < a->nCells; c++) {
        double out = 0.0;
        for (int f = a->ownerStart[c]; f < a->ownerStart[c + 1]; f++)
            out = out + A->upper[f] * psi[a->u[f]];
        for (int k = a->losortStart[c]; k < a->losortStart[c + 1]; k++) {
            int f = a->losort[k];
            out = out + A->lower[f] * psi[a->l[f]];
        }
        Apsi[c] = out;
    }
    if (pnf) { /* updateMatrixInterfaces: Apsi[cell] -= bou*psiNbr */
        int tot = a->patchStart[a->nPatches];
        for (int i = 0; i < tot; i++) {
            double v = A->bou[i] * pnf[i];
            Apsi[a->faceCells[i]] = Apsi[a->faceCells[i]] + (-v);
        }
        free(pnf);
    }
    for (int c = 0; c < a->nCells; c++) psi[c] = -Apsi[c] / A->diag[c];
}

/* dense LU with partial pivoting of the coarsest matrix, standing in for
 * matrices/LUscalarMatrix (GAMGSolver.C:144-172, GAMGSolverSolve.C:564-569).  With more
 * than one rank the coarsest matrices of all ranks (and their processor-interface
 * coefficients, LUscalarMatrix.C:201-270: A[row][col of the neighbour cell] -= coeff) are
 * assembled into one global matrix; every rank factorises the same matrix. */
typedef struct {
    int n;        /* global size */
    int nLocal, offset, nMax, nRanks;
    double *lu;
    int *piv;
} dense_lu;

/* LUDecompose: matrices/scalarMatrices/scalarMatrices.C:42-146 -- Crout's method with implicit
 * (row-scaled) partial pivoting; a later row wins a tie (`>=`), a zero pivot becomes SMALL = 1e-15. */
static void lu_factor_inplace(dense_lu *d)
{
    int n = d->n;
    double *A = d->lu;
    double *vv = (double *)malloc(sizeof(double) * (size_t)(n > 0 ? n : 1));
    for (int i = 0; i < n; i++) {
        double largest = 0.0;
        for (int j = 0; j < n; j++) {
            double t = fabs(A[(size_t)i * n + j]);
            if (t > largest) largest = t;
        }
        vv[i] = 1.0 / largest; /* the reference aborts on a zero row ("Singular matrix") */
    }
    for (int j = 0; j < n; j++) {
        for (int i = 0; i < j; i++) {
            double sum = A[(size_t)i * n + j];
            for (int k = 0; k < i; k++) sum -= A[(size_t)i * n + k] * A[(size_t)k * n + j];
            A[(size_t)i * n + j] = sum;
        }
        int iMax = 0;
        double largest = 0.0;
        for (int i = j; i < n; i++) {
            double sum = A[(size_t)i * n + j];
            for (int k = 0; k < j; k++) sum -= A[(size_t)i * n + k] * A[(size_t)k * n + j];
            A[(size_t)i * n + j] = sum;
            double t = vv[i] * fabs(sum);
            if (t >= largest) {
                largest = t;
                iMax = i;
            }
        }
        d->piv[j] = iMax;
        if (j != iMax) {
            for (int k = 0; k < n; k++) {
                double t = A[(size_t)j * n + k];
                A[(size_t)j * n + k] = A[(size_t)iMax * n + k];
                A[(size_t)iMax * n + k] = t;
            }
            vv[iMax] = vv[j];
        }
        if (A[(size_t)j * n + j] == 0.0) A[(size_t)j * n + j] = 1.0e-15;
        if (j != n - 1) {
            double rDiag = 1.0 / A[(size_t)j * n + j];
            for (int i = j + 1; i < n; i++) A[(size_t)i * n + j] *= rDiag;
        }
    }
    free(vv);
}

static dense_lu *lu_factor(const orc_matrix *A, const orc_comm *comm)
{
    const orc_addr *a = A->a;
    int nl = a->nCells;
    dense_lu *d = (dense_lu *)calloc(1, sizeof(dense_lu));
    int R = (comm && comm->gather && comm->nRanks > 1) ? comm->nRanks : 1;
    d->nRanks = R;
    d->nLocal = nl;
    int *counts = (int *)calloc((size_t)R, sizeof(int));
    if (R > 1) {
        double mine = nl;
        double *all = (double *)calloc((size_t)R, sizeof(double));
        comm->gather(comm->ctx, &mine, 1, all);
        for (int r = 0; r < R; r++) counts[r] = (int)all[r];
        free(all);
    } else
        counts[0] = nl;
    int N = 0, nMax = 0, *offs = (int *)calloc((size_t)R + 1, sizeof(int));
    for (int r = 0; r < R; r++) {
        offs[r] = N;
        N += counts[r];
        if (counts[r] > nMax) nMax = counts[r];
    }
    int me = R > 1 ? comm->rank : 0;
    d->n = N;
    d->offset = offs[me];
    d->nMax = nMax;
    /* local rows of the global matrix */
    double *rows = (double *)calloc((size_t)nMax * N, sizeof(double));
    for (int c = 0; c < nl; c++) rows[(size_t)c * N + offs[me] + c] = A->diag[c];
    for (int f = 0; f < a->nFaces; f++) {
        rows[(size_t)a->l[f] * N + offs[me] + a->u[f]] += A->upper[f];
        rows[(size_t)a->u[f] * N + offs[me] + a->l[f]] += A->lower[f];
    }
    if (a->nPatches && a->neighbRank) { /* coupled patches: processor (another rank's columns) or cyclic (this rank's) */
        double *ids = (double *)malloc(sizeof(double) * (size_t)nl);
        for (int c = 0; c < nl; c++) ids[c] = (double)c;
        double *nbrCell = orc_halo_exchange(a, ids, comm);
        free(ids);
        for (int p = 0; p < a->nPatches; p++) {
            int nbRank = a->neighbRank[p] >= 0 ? a->neighbRank[p] : me;
            if (nbRank != me && R == 1) continue;
            for (int i = a->patchStart[p]; i < a->patchStart[p + 1]; i++)
                rows[(size_t)a->faceCells[i] * N + offs[nbRank] + (int)nbrCell[i]] -= A->bou[i];
        }
        free(nbrCell);
    }
    d->lu = (double *)calloc((size_t)N * N, sizeof(double));
    if (R > 1) {
        double *all = (double *)calloc((size_t)R * nMax * N, sizeof(double));
        comm->gather(comm->ctx, rows, nMax * N, all);
        for (int r = 0; r < R; r++)
            for (int i = 0; i < counts[r]; i++)
                memcpy(d->lu + (size_t)(offs[r] + i) * N, all + ((size_t)r * nMax + i) * N, sizeof(double) * (size_t)N);
        free(all);
    } else
        memcpy(d->lu, rows, sizeof(double) * (size_t)N * N);
    free(rows);
    d->piv = (int *)malloc(sizeof(int) * (size_t)N);
    /* keep counts/offs for the per-cycle gather */
    d->piv = (int *)realloc(d->piv, sizeof(int) * ((size_t)N + 2 * (size_t)R + 2));
    memcpy(d->piv + N, counts, sizeof(int) * (size_t)R);
    memcpy(d->piv + N + R, offs, sizeof(int) * ((size_t)R + 1));
    free(counts);
    free(offs);
    lu_factor_inplace(d);
    return d;
}

/* x (local part) = (A_global^-1 b_global)(local part) */
static void lu_solve(const dense_lu *d, const double *bLocal, double *xLocal, const orc_comm *comm)
{
    int n = d->n, R = d->nRanks;
    const int *counts = d->piv + n, *offs = d->piv + n + R;
    double *b = (double *)calloc((size_t)n, sizeof(double));
    if (R > 1) {
        double *mine = (double *)calloc((size_t)d->nMax, sizeof(double));
        double *all = (double *)calloc((size_t)R * d->nMax, sizeof(double));
        memcpy(mine, bLocal, sizeof(double) * (size_t)d->nLocal);
        comm->gather(comm->ctx, mine, d->nMax, all);
        for (int r = 0; r < R; r++) memcpy(b + offs[r], all + (size_t)r * d->nMax, sizeof(double) * (size_t)counts[r]);
        free(mine);
        free(all);
    } else
        memcpy(b, bLocal, sizeof(double) * (size_t)n);
    /* LUBacksubstitute: scalarMatricesTemplates.C:119-164 (forward pass skips the leading zeros of b) */
    int ii = 0;
    for (int i = 0; i < n; i++) {
        int ip = d->piv[i];
        double sum = b[ip];
        b[ip] = b[i];
        if (ii != 0) {
            for (int j = ii - 1; j < i; j++) sum -= d->lu[(size_t)i * n + j] * b[j];
        } else if (sum != 0.0) {
            ii = i + 1;
        }
        b[i] = sum;
    }
    for (int i = n - 1; i >= 0; i--) {
        double sum = b[i];
        for (int j = i + 1; j < n; j++) sum -= d->lu[(size_t)i * n + j] * b[j];
        b[i] = sum / d->lu[(size_t)i * n + i];
    }
    memcpy(xLocal, b + d->offset, sizeof(double) * (size_t)d->nLocal);
    free(b);
}

void orc_gamg_set_coarsest_inverse(orc_gamg *g, const double *invRows, const int *perm, int N)
{
    free(g->devInv);
    free(g->devPerm);
    g->devInv = NULL;
    g->devPerm = NULL;
    g->devN = 0;
    if (!invRows || g->nLevels == 0) return;
    int n = g->addr[g->nLevels - 1]->nCells;
    g->devN = N;
    g->devInv = (double *)malloc(sizeof(double) * ((size_t)n * N + 1));
    g->devPerm = (int *)malloc(sizeof(int) * ((size_t)n + 1));
    memcpy(g->devInv, invRows, sizeof(double) * (size_t)n * N);
    memcpy(g->devPerm, perm, sizeof(int) * (size_t)n);
}

void orc_gamg_set_scale_order(orc_gamg *g, int descending) { g->scaleDescending = descending; }

/* x[c] = sum_j inv[perm[c]][j] * bg[j] with bg the right-hand sides of all ranks in banded order (rank offset +
 * banded row), one fused multiply-add per term in ascending j from zero */
static void dev_inverse_apply(const orc_gamg *g, int n, const double *b, double *x, const orc_comm *comm)
{
    int N = g->devN, R = (comm && comm->gather && comm->nRanks > 1) ? comm->nRanks : 1;
    double *bg = (double *)calloc((size_t)N + 1, sizeof(double));
    if (R > 1) {
        double mine = n, *cnt = (double *)calloc((size_t)R, sizeof(double));
        comm->gather(comm->ctx, &mine, 1, cnt);
        int nMax = 0;
        for (int r = 0; r < R; r++) nMax = (int)cnt[r] > nMax ? (int)cnt[r] : nMax;
        double *bb = (double *)calloc((size_t)nMax + 1, sizeof(double));
        double *all = (double *)calloc((size_t)R * nMax + 1, sizeof(double));
        for (int c = 0; c < n; c++) bb[g->devPerm[c]] = b[c];
        comm->gather(comm->ctx, bb, nMax, all);
        for (int r = 0, o = 0; r < R; o += (int)cnt[r], r++)
            memcpy(bg + o, all + (size_t)r * nMax, sizeof(double) * (size_t)cnt[r]);
        free(cnt);
        free(bb);
        free(all);
    } else
        for (int c = 0; c < n; c++) bg[g->devPerm[c]] = b[c];
    for (int c = 0; c < n; c++) {
        const double *row = g->devInv + (size_t)g->devPerm[c] * N;
        double s = 0.0;
        for (int j = 0; j < N; j++) s = fma(row[j], bg[j], s);
        x[c] = s;
    }
    free(bg);
}

/* the coarse matrix of level lev for the finest matrix m, as the solve builds it */
void orc_gamg_coarse_matrix(const orc_matrix *m, const orc_gamg *g, int lev, double *diag, double *upper,
                            double *lower, double *bou, double *intc)
{
    lev_matrix *lm = (lev_matrix *)calloc((size_t)lev + 1, sizeof(lev_matrix));
    for (int k = 0; k <= lev; k++) {
        const double *fd = k ? lm[k - 1].diag : m->diag;
        const double *fu = k ? lm[k - 1].upper : m->upper;
        const double *fl = k ? lm[k - 1].lower : (m->symmetric ? NULL : m->lower);
        const double *fb = k ? lm[k - 1].bou : m->bou;
        const double *fi = k ? lm[k - 1].intc : m->intc;
        agglomerate_matrix(g, k, fd, fu, fl, fb, fi, &lm[k]);
    }
    const lev_matrix *L = &lm[lev];
    int nCP = orc_gamg_npatchfaces(g, lev);
    memcpy(diag, L->diag, sizeof(double) * (size_t)L->n);
    memcpy(upper, L->upper, sizeof(double) * (size_t)L->nf);
    if (lower && L->lower) memcpy(lower, L->lower, sizeof(double) * (size_t)L->nf);
    if (bou) memcpy(bou, L->bou, sizeof(double) * (size_t)nCP);
    if (intc) memcpy(intc, L->intc, sizeof(double) * (size_t)nCP);
    for (int k = 0; k <= lev; k++) {
        free(lm[k].diag);
        free(lm[k].upper);
        free(lm[k].lower);
        free(lm[k].bou);
        free(lm[k].intc);
        orc_matrix_free(lm[k].m);
    }
    free(lm);
}

static int imin(int a, int b) { return a < b ? a : b; }

/* GAMGSolver::solve + Vcycle: GAMGSolverSolve.C:59-474 */
int orc_gamg_solve(const orc_matrix *m, orc_gamg *g, const char *smoother, const orc_controls *c,
                   double *psi, const double *source, const orc_comm *comm, orc_perf *perf, double *hist,
                   int histCap)
{
    memset(perf, 0, sizeof(*perf));
    strcpy(perf->solverName, "GAMG");
    if (smoother && *smoother && strcmp(smoother, "Jacobi") && strcmp(smoother, "GaussSeidel"))
        return -2; /* GaussSeidel aliases to Jacobi: GaussSeidelSmoother.C:43-69 */
    int nL = g->nLevels;
    if (nL == 0) return -4; /* GAMGSolver.C:174-192 "No coarse levels created" */
    int n = m->a->nCells;
    int scaleCorrection = c->scaleCorrection < 0 ? m->symmetric : c->scaleCorrection;
    double tol = c->tolerance, relTol = c->relTol;

    /* constructor: coarse matrices for every level (GAMGSolver.C:85-96) */
    lev_matrix *lm = (lev_matrix *)calloc((size_t)nL, sizeof(lev_matrix));
    for (int lev = 0; lev < nL; lev++) {
        const double *fd = lev ? lm[lev - 1].diag : m->diag;
        const double *fu = lev ? lm[lev - 1].upper : m->upper;
        const double *fl = lev ? lm[lev - 1].lower : (m->symmetric ? NULL : m->lower);
        const double *fb = lev ? lm[lev - 1].bou : m->bou;
        const double *fi = lev ? lm[lev - 1].intc : m->intc;
        agglomerate_matrix(g, lev, fd, fu, fl, fb, fi, &lm[lev]);
    }
    int coarsest = nL - 1;
    dense_lu *lu = c->directSolveCoarsest && !g->devInv ? lu_factor(lm[coarsest].m, comm) : NULL;

    double *Apsi = (double *)calloc((size_t)n, sizeof(double));
    double *finestCorr = (double *)calloc((size_t)n, sizeof(double));
    double *finestRes = (double *)calloc((size_t)n, sizeof(double));
    orc_amul(m, psi, Apsi, comm);
    double normFactor = orc_normFactor(m, psi, source, Apsi, finestCorr, comm);
    perf->normFactor = normFactor;
    for (int i = 0; i < n; i++) finestRes[i] = source[i] - Apsi[i];
    perf->initialResidual = orc_gsummag(finestRes, n, comm) / normFactor;
    perf->finalResidual = perf->initialResidual;
    if (hist && histCap > 0) hist[0] = perf->finalResidual;

#define CONVERGED()                                                                        \
    (perf->converged = (perf->finalResidual < tol ||                                       \
                        (relTol > 1e-20 && perf->finalResidual < relTol * perf->initialResidual)))

    if (c->minIter > 0 || !CONVERGED()) {
        double **corr = (double **)calloc((size_t)nL, sizeof(double *));
        double **src = (double **)calloc((size_t)nL, sizeof(double *));
        int maxSize = n;
        for (int lev = 0; lev < nL; lev++) {
            corr[lev] = (double *)calloc((size_t)(lm[lev].n > 0 ? lm[lev].n : 1), sizeof(double));
            src[lev] = (double *)calloc((size_t)(lm[lev].n > 0 ? lm[lev].n : 1), sizeof(double));
            if (lm[lev].n > maxSize) maxSize = lm[lev].n;
        }
        double *scratch1 = (double *)calloc((size_t)maxSize, sizeof(double));
        double *scratch2 = (double *)calloc((size_t)maxSize, sizeof(double));
        do {
            /* ---- Vcycle :181-474 ---- */
            restrict_field(g->restrictAddr[0], n, lm[0].n, finestRes, src[0]);
            for (int lev = 0; lev < coarsest; lev++) {
                if (c->nPreSweeps) {
                    memset(corr[lev], 0, sizeof(double) * (size_t)lm[lev].n);
                    orc_jacobi_smooth(lm[lev].m, c->omega, corr[lev], src[lev],
                                      imin(c->nPreSweeps + c->preSweepsLevelMultiplier * lev,
                                           c->maxPreSweeps),
                                      comm);
                    double *ACf = scratch1;
                    if (scaleCorrection && lev < coarsest - 1)
                        gamg_scale(lm[lev].m, corr[lev], ACf, src[lev], comm, g->scaleDescending);
                    orc_amul(lm[lev].m, corr[lev], ACf, comm);
                    for (int i = 0; i < lm[lev].n; i++) src[lev][i] -= ACf[i];
                }
                restrict_field(g->restrictAddr[lev + 1], lm[lev].n, lm[lev + 1].n, src[lev],
                               src[lev + 1]);
            }
            /* solveCoarsestLevel :552-619 */
            if (c->directSolveCoarsest && g->devInv) {
                dev_inverse_apply(g, lm[coarsest].n, src[coarsest], corr[coarsest], comm);
            } else if (c->directSolveCoarsest) {
                lu_solve(lu, src[coarsest], corr[coarsest], comm);
            } else {
                orc_controls cc;
                orc_controls_default(&cc);
                cc.tolerance = tol;
                cc.relTol = relTol;
                orc_perf cp;
                memset(corr[coarsest], 0, sizeof(double) * (size_t)lm[coarsest].n);
                orc_solve(lm[coarsest].m, lm[coarsest].lower ? "BICCG" : "ICCG", NULL, &cc,
                          corr[coarsest], src[coarsest], comm, &cp, NULL, 0);
            }
            for (int lev = coarsest - 1; lev >= 0; lev--) {
                double *pre = scratch2;
                if (c->nPreSweeps) memcpy(pre, corr[lev], sizeof(double) * (size_t)lm[lev].n);
                prolong_field(g->restrictAddr[lev + 1], lm[lev].n, corr[lev + 1], corr[lev]);
                double *ACf = scratch1;
                if (c->interpolateCorrection) gamg_interpolate(lm[lev].m, corr[lev], ACf, comm);
                if (scaleCorrection && (c->interpolateCorrection || lev < coarsest - 1))
                    gamg_scale(lm[lev].m, corr[lev], ACf, src[lev], comm, g->scaleDescending);
                if (c->nPreSweeps)
                    for (int i = 0; i < lm[lev].n; i++) corr[lev][i] += pre[i];
                orc_jacobi_smooth(lm[lev].m, c->omega, corr[lev], src[lev],
                                  imin(c->nPostSweeps + c->postSweepsLevelMultiplier * lev,
                                       c->maxPostSweeps),
                                  comm);
            }
            prolong_field(g->restrictAddr[0], n, corr[0], finestCorr);
            if (c->interpolateCorrection) gamg_interpolate(m, finestCorr, Apsi, comm);
            if (scaleCorrection) gamg_scale(m, finestCorr, Apsi, finestRes, comm, g->scaleDescending);
            for (int i = 0; i < n; i++) psi[i] = psi[i] + finestCorr[i];
            orc_jacobi_smooth(m, c->omega, psi, source, c->nFinestSweeps, comm);
            /* ---- end Vcycle ---- */
            orc_amul(m, psi, Apsi, comm);
            for (int i = 0; i < n; i++) finestRes[i] = source[i] - Apsi[i];
            perf->finalResidual = orc_gsummag(finestRes, n, comm) / normFactor;
            if (hist && perf->nIterations + 1 < histCap) hist[perf->nIterations + 1] = perf->finalResidual;
        } while ((++perf->nIterations < c->maxIter && !CONVERGED()) ||
                 perf->nIterations < c->minIter);
        for (int lev = 0; lev < nL; lev++) {
            free(corr[lev]);
            free(src[lev]);
        }
        free(corr);
        free(src);
        free(scratch1);
        free(scratch2);
    }
#undef CONVERGED
    if (lu) {
        free(lu->lu);
        free(lu->piv);
        free(lu);
    }
    for (int lev = 0; lev < nL; lev++) {
        free(lm[lev].diag);
        free(lm[lev].upper);
        free(lm[lev].lower);
        free(lm[lev].bou);
        free(lm[lev].intc);
        orc_matrix_free(lm[lev].m);
    }
    free(lm);
    free(Apsi);
    free(finestCorr);
    free(finestRes);
    return 0;
}
