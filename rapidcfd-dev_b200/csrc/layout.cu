// layout.cu -- host-side construction of the banded block layout ("warp-contiguous
// bands") from OpenFOAM lduAddressing.  Replaces the reference's derived addressing
// (LDU/lduAddressing/lduAddressing.C:169-400: losort, ownerStart, losortStart,
// ownerSortAddr, patchSort*) and lduMatrix::calcSortCoeffs (LDU/lduMatrix/lduMatrix.C:380-471).
//
// Design (DESIGN.md section 3):
//  * cells are renumbered so that BAND_ROWS consecutive rows form a spatially compact
//    brick (Morton order over power-of-two tiles of the cell-centre bounding box, caller
//    order inside a tile; without centres a graph-distance embedding stands in);
//  * every row keeps its entries in the reference's summation order (owner faces by
//    face index, neighbour faces in losort order, coupled-patch faces in patch order);
//  * entries of 64 consecutive rows are stored slot-major ("slice"): slot j of row q
//    sits at sliceStart + 64*j + q, so a warp reads one slot of its 64 rows with a
//    single 128-bit load per lane;
//  * columns are 16-bit indices into the band's shared-memory psi tile: the band's own
//    rows first, then the band's halo list (rows of other bands / received interface
//    values) which is gathered once per band.
//
// layout_build runs in stages: addressing checks and CSR, renumbering, coupled-patch face
// lists, then a plan for a band size (halved until the band fits), the face-stream choice,
// and the fills of the entry stream and (where it is used) the face stream and its template table.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <numeric>
#include <queue>
#include <unordered_map>

#include "internal.h"

namespace {

// the addressing seen from both sides of every face, and each cell's coupled-patch faces
struct Graph {
    int nCells, nFaces, nRecv;
    const std::vector<int> &l, &u;
    std::vector<int> ownerStart, losortStart, losort;
    std::vector<int> pfStart, pfItem; // cell -> coupled-patch faces, in (patch, patch face) order
};

// cell -> faces it owns is contiguous (faces sorted by owner); cell -> faces where it is neighbour is the stable
// counting sort the reference calls losort (csr_from_map of the neighbours)
void build_owner_start(int nCells, const std::vector<int> &l, std::vector<int> &ownerStart)
{
    ownerStart.assign((size_t)nCells + 1, 0);
    for (size_t f = 0; f < l.size(); f++) ownerStart[l[f] + 1]++;
    for (int c = 0; c < nCells; c++) ownerStart[c + 1] += ownerStart[c];
}

// breadth-first graph distance from `seed` (used when no cell centres are given);
// further components, if any, restart from their lowest cell
void bfs_dist(const Graph &g, int seed, std::vector<int> &dist)
{
    dist.assign(g.nCells, -1);
    std::vector<int> q;
    q.reserve(g.nCells);
    auto grow = [&](int s) {
        size_t head = q.size();
        dist[s] = 0;
        q.push_back(s);
        while (head < q.size()) {
            int c = q[head++];
            for (int f = g.ownerStart[c]; f < g.ownerStart[c + 1]; f++)
                if (dist[g.u[f]] < 0) {
                    dist[g.u[f]] = dist[c] + 1;
                    q.push_back(g.u[f]);
                }
            for (int k = g.losortStart[c]; k < g.losortStart[c + 1]; k++) {
                int nb = g.l[g.losort[k]];
                if (dist[nb] < 0) {
                    dist[nb] = dist[c] + 1;
                    q.push_back(nb);
                }
            }
        }
    };
    grow(seed);
    for (int c = 0; c < g.nCells; c++)
        if (dist[c] < 0) grow(c);
}

int argmax(const std::vector<int> &v)
{
    return (int)(std::max_element(v.begin(), v.end()) - v.begin());
}

uint64_t interleave(const uint32_t idx[3], const int bits[3])
{
    // axis 0 provides the lowest bit of each round so that consecutive tiles are
    // x-neighbours first
    uint64_t code = 0;
    int pos = 0;
    int maxb = std::max(bits[0], std::max(bits[1], bits[2]));
    for (int b = 0; b < maxb; b++)
        for (int ax = 0; ax < 3; ax++)
            if (b < bits[ax]) code |= (uint64_t)((idx[ax] >> b) & 1u) << pos++;
    return code;
}

// a band's tile is (bandRows + halo) doubles of the one staged vector (engine.cuh); H100 gives a CTA up to 227 KB,
// the kernel keeps a little static scratch
constexpr size_t TILE_BYTES_MAX = 200 * 1024;

int pick_band_rows(int nCells, int smCount, int packCtas)
{
    if (const char *e = getenv("B200LDU_BAND_ROWS")) {
        int v = atoi(e);
        if (v >= SLICE_ROWS && v % SLICE_ROWS == 0 && v <= 16384) return v;
    }
    // A sweep is one CTA per band, 6 resident per SM (792 slots on an H100 with 132 SMs).  Measured on one H100 80GB HBM3
    // (400 W power limit), bench.py --steps 20, Mcell-iters/s with matrix_set, one sample each:
    //   128^3:  512 rows (this rule) 9.9 k | 1024 rows 9.8 k | 2048 rows 9.2 k | 2688 rows (one wave, 781 CTAs) 9.0 k
    //   256^3: 1024 rows 10.4 k | 2048 rows 9.9 k | 2688 rows 9.3 k
    // and at a 700 W power limit, 256^3, alternating runs: 1024 rows (this rule) 11.66-11.68 k (3 runs) | 2048 rows 11.01 k (4 runs).
    // A mesh that fits one wave is best served by exactly one (every CTA resident at once, fewer partial sums for
    // the scalar step).  Beyond that, whole waves are the WORST choice -- the CTAs of a wave stage and stream in lock-step, so the
    // SM alternates between a latency-bound and a bandwidth-bound phase -- and 4+ waves of smaller bands, which drift out of
    // phase, are best.  At 256^3 a 1024-row band's sweep A (the AINV sweep, whose staging phase carries most of its
    // vector bytes) takes 782 us against 849 us for 2048 rows; sweep B 583 against 597 us (torch.profiler,
    // bench_kernels.py --pcg-sweeps): 20 waves drift apart better than 10.
    // The bands grow to 512 rows as the mesh allows: there the face stream of symmetric matrices (tile + product buffer,
    // ~23 KB) keeps 6 CTAs per SM, at 1024 rows (~46 KB) only 4.  Measured on one H100 80GB HBM3 at a 400 W power
    // limit, 256^3, bench.py --steps 5, three alternating runs each: 512 rows + face stream (this rule) 12.44-12.51 k |
    // 1024 rows + face stream 11.88-11.89 k | 1024 rows, entry stream (the previous rule) 11.23-11.27 k.  The
    // asymmetric PBiCG leg, which keeps the entry stream, loses 1.4 % to the narrower bands (5.57-5.58 k against
    // 5.65-5.66 k).
    // the packing CTAs of the fused halo send share the grid with the bands: keep bands + packers within the one wave
    const long long slots = (long long)(smCount > 0 ? smCount : 132) * 6 - packCtas;
    const long long maxRows = 2432; // the tile of a band + its halo must leave room for 6 CTAs per SM
    if (nCells <= slots * maxRows) {
        const long long perBand = (nCells + slots - 1) / slots;
        long long rows = ((perBand + SLICE_ROWS - 1) / SLICE_ROWS) * SLICE_ROWS;
        return (int)std::max<long long>(rows, SLICE_ROWS);
    }
    const long long target = nCells / (slots * 4);
    int b = SLICE_ROWS;
    while (b * 2 <= target && b < 512) b *= 2;
    return b;
}

// resident engine CTAs per SM for a band's dynamic shared memory: 228 KB per SM, 1 KB of it reserved per CTA and
// about 1 KB of static scratch; the 40-register budget allows 6
int ctas_per_sm(long long smemDoubles)
{
    const long long per = smemDoubles * (long long)sizeof(double) + 2048;
    return (int)std::min<long long>(6, 228 * 1024 / per);
}

// ---- 1. addressing checks and CSR --------------------------------------------
int build_csr(Graph &g)
{
    if (g.nCells <= 0) {
        b200_set_error("layout_build: nCells must be positive");
        return B200LDU_EINVAL;
    }
    for (int f = 0; f < g.nFaces; f++) {
        if (g.l[f] < 0 || g.u[f] >= g.nCells || g.l[f] >= g.u[f] || (f && g.l[f] < g.l[f - 1])) {
            b200_set_error("layout_build: face %d violates upper-triangular owner-sorted order", f);
            return B200LDU_EINVAL;
        }
    }
    build_owner_start(g.nCells, g.l, g.ownerStart);
    csr_from_map(g.u, g.nCells, g.losortStart, g.losort);
    return B200LDU_OK;
}

// ---- 2. cell renumbering: banded row -> caller cell, whatever the band size ----
std::vector<int> renumber(const Graph &g, const double *centres)
{
    const int nCells = g.nCells;
    std::vector<double> emb; // 3 coordinates per cell
    const double *xyz = centres;
    if (!xyz) {
        std::vector<int> d0, d1, d2, d3;
        bfs_dist(g, 0, d0);
        int s1 = argmax(d0);
        bfs_dist(g, s1, d1);
        int s2 = argmax(d1);
        bfs_dist(g, s2, d2);
        std::vector<int> sum(nCells);
        for (int c = 0; c < nCells; c++) sum[c] = d1[c] + d2[c];
        int s3 = argmax(sum);
        bfs_dist(g, s3, d3);
        emb.resize((size_t)3 * nCells);
        for (int c = 0; c < nCells; c++) {
            emb[3 * (size_t)c + 0] = d1[c];
            emb[3 * (size_t)c + 1] = d2[c];
            emb[3 * (size_t)c + 2] = d3[c];
        }
        xyz = emb.data();
    }
    double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300};
    for (int c = 0; c < nCells; c++)
        for (int k = 0; k < 3; k++) {
            double v = xyz[3 * (size_t)c + k];
            lo[k] = std::min(lo[k], v);
            hi[k] = std::max(hi[k], v);
        }
    double ext[3];
    for (int k = 0; k < 3; k++) ext[k] = std::max(hi[k] - lo[k], 1e-300);
    int bits[3] = {0, 0, 0};
    {
        long long tiles = 1;
        // tiles of ~one slice (64 rows): slices become small cubes (most of a row's faces stay inside its slice) and Morton order keeps
        // every run of bandRows/64 consecutive tiles a compact brick
        while ((double)nCells / (double)tiles > (double)SLICE_ROWS && bits[0] + bits[1] + bits[2] < 45) {
            int best = 2; // ties go to the last axis so x keeps the longest runs
            double bestExt = -1;
            for (int k = 2; k >= 0; k--) {
                double e = ext[k] / (double)(1 << bits[k]);
                if (e > bestExt * (1 + 1e-9)) {
                    bestExt = e;
                    best = k;
                }
            }
            bits[best]++;
            tiles *= 2;
        }
    }
    std::vector<uint64_t> key(nCells);
#pragma omp parallel for schedule(static)
    for (int c = 0; c < nCells; c++) {
        uint32_t idx[3];
        for (int k = 0; k < 3; k++) {
            double t = (xyz[3 * (size_t)c + k] - lo[k]) / ext[k];
            long long q = (long long)(t * (double)(1 << bits[k]));
            long long mx = (1ll << bits[k]) - 1;
            idx[k] = (uint32_t)std::min(std::max(q, 0ll), mx);
        }
        key[c] = interleave(idx, bits);
    }
    std::vector<int> order(nCells);
    int kb = bits[0] + bits[1] + bits[2];
    if (kb <= 26) { // counting sort (stable => caller order inside a tile)
        size_t nT = (size_t)1 << kb;
        std::vector<int> cnt(nT + 1, 0);
        for (int c = 0; c < nCells; c++) cnt[key[c] + 1]++;
        for (size_t t = 0; t < nT; t++) cnt[t + 1] += cnt[t];
        for (int c = 0; c < nCells; c++) order[cnt[key[c]]++] = c;
    } else {
        std::iota(order.begin(), order.end(), 0);
        std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return key[x] < key[y]; });
    }
    return order;
}

// ---- 3. cell -> coupled-patch faces: csr_from_map of the face cells (layout_build) ----

// ---- 4. plan for one band size --------------------------------------------------
// Everything but the two streams' entries: slice widths and offsets of both streams, the face stream's list bounds,
// the per-band halo lists and whether the band fits.
struct Plan {
    LayoutHost H;
    std::vector<int> iperm;             // [nPad] banded row -> caller cell, -1 padding
    std::vector<std::vector<int>> halo; // per band: extended indices of its outside columns, sorted
    int tooWide = 0;                    // bands with more than 65535 tile columns
    bool tileFits = false;              // the tile of every band fits in shared memory
    bool fsFits = false;                // the 16-bit product slots address the buffer, the 32-bit offsets every entry
};

int plan_layout(const Graph &g, const std::vector<int> &order, const std::vector<int> &perm, int bandRows, Plan &P)
{
    P = Plan{};
    LayoutHost &H = P.H;
    const int nBands = (g.nCells + bandRows - 1) / bandRows;
    const int nPad = nBands * bandRows;
    const int slicesPerBand = bandRows / SLICE_ROWS;
    const int nSlices = nPad / SLICE_ROWS;
    H.nPad = nPad;
    H.nBands = nBands;
    H.bandRows = bandRows;
    H.nRecv = g.nRecv;
    P.iperm = order;
    P.iperm.resize(nPad, -1);
    const std::vector<int> &iperm = P.iperm;

    // slice widths: entry stream (owner + neighbour entries, then interfaces) and face stream (owner entries; buffer
    // slots for neighbour and interface products)
    H.sliceW.assign(nSlices, 0);
    H.sliceWL.assign(nSlices, 0);
    H.fsSlice.assign(nSlices, FsSlice{});
    int bad = 0;
#pragma omp parallel for schedule(static) reduction(+ : bad)
    for (int s = 0; s < nSlices; s++) {
        int wl = 0, wo = 0, wn = 0, wi = 0;
        for (int q = 0; q < SLICE_ROWS; q++) {
            int c = iperm[(size_t)s * SLICE_ROWS + q];
            if (c < 0) continue;
            const int no = g.ownerStart[c + 1] - g.ownerStart[c], nn = g.losortStart[c + 1] - g.losortStart[c];
            wl = std::max(wl, no + nn);
            wo = std::max(wo, no);
            wn = std::max(wn, nn);
            wi = std::max(wi, g.pfStart[c + 1] - g.pfStart[c]);
        }
        if (wl + wi > 65535) bad++;
        H.sliceWL[s] = (uint16_t)wl;
        H.sliceW[s] = (uint16_t)(wl + wi);
        H.fsSlice[s] = FsSlice{0, 0, 0, (uint16_t)wo, (uint16_t)wn, (uint16_t)wi};
    }
    if (bad) {
        b200_set_error("layout_build: a row has more than 65535 entries");
        return B200LDU_ELAYOUT;
    }
    H.sliceStart.assign((size_t)nSlices + 1, 0);
    for (int s = 0; s < nSlices; s++)
        H.sliceStart[s + 1] = H.sliceStart[s] + (long long)H.sliceW[s] * SLICE_ROWS;
    H.nEntries = H.sliceStart[nSlices];

    // face stream: owner-stream and product-buffer offsets of each slice, then the list bounds of each band
    long long fsOwn = 0;
    for (int b = 0; b < nBands; b++) {
        long long off = 0;
        for (int sl = 0; sl < slicesPerBand; sl++) {
            FsSlice &S = H.fsSlice[(size_t)b * slicesPerBand + sl];
            S.start64 = (int)(fsOwn / SLICE_ROWS);
            S.bufOff = (uint16_t)std::min<long long>(off, 0xffff); // exact where the face stream fits (fsFits)
            fsOwn += (long long)S.wo * SLICE_ROWS;
            off += (1 + (long long)S.wn + S.wi) * SLICE_ROWS;
        }
        H.fsBufMax = std::max(H.fsBufMax, off);
    }
    std::vector<int> &fsListStart = H.fsListStart, &fsListIfc = H.fsListIfc;
    fsListStart.assign((size_t)nBands + 1, 0); // counts first
    fsListIfc.assign(nBands, 0);
#pragma omp parallel for schedule(static)
    for (int b = 0; b < nBands; b++) {
        const int r0 = b * bandRows, r1 = r0 + bandRows;
        int nx = 0, ni = 0;
        for (int r = r0; r < r1; r++) {
            int c = iperm[r];
            if (c < 0) continue;
            for (int k = g.losortStart[c]; k < g.losortStart[c + 1]; k++) {
                int t = perm[g.l[g.losort[k]]];
                nx += (t < r0 || t >= r1);
            }
            ni += g.pfStart[c + 1] - g.pfStart[c];
        }
        fsListIfc[b] = nx;
        fsListStart[b + 1] = nx + ni;
    }
    fsListStart[0] = (int)std::min<long long>(fsOwn, INT32_MAX);
    for (int b = 0; b < nBands; b++) {
        const long long next = (long long)fsListStart[b] + fsListStart[b + 1];
        fsListIfc[b] += fsListStart[b];
        fsListStart[b + 1] = (int)std::min<long long>(next, INT32_MAX);
    }
    H.fsOwn = fsOwn;
    H.fsList = (long long)fsListStart[nBands] - fsListStart[0];
    P.fsFits = H.fsBufMax < (long long)FS_PAD && H.fsOwn + H.fsList < INT32_MAX;

    // per-band halo lists
    P.halo.resize(nBands);
    int tooWide = 0;
#pragma omp parallel for schedule(dynamic, 4) reduction(+ : tooWide)
    for (int b = 0; b < nBands; b++) {
        const int r0 = b * bandRows, r1 = r0 + bandRows;
        std::vector<int> &h = P.halo[b];
        for (int r = r0; r < r1; r++) {
            int c = iperm[r];
            if (c < 0) continue;
            for (int f = g.ownerStart[c]; f < g.ownerStart[c + 1]; f++) {
                int t = perm[g.u[f]];
                if (t < r0 || t >= r1) h.push_back(t);
            }
            for (int k = g.losortStart[c]; k < g.losortStart[c + 1]; k++) {
                int t = perm[g.l[g.losort[k]]];
                if (t < r0 || t >= r1) h.push_back(t);
            }
            for (int k = g.pfStart[c]; k < g.pfStart[c + 1]; k++) h.push_back(nPad + g.pfItem[k]);
        }
        std::sort(h.begin(), h.end());
        h.erase(std::unique(h.begin(), h.end()), h.end());
        if ((long long)bandRows + (long long)h.size() > 65536) tooWide++;
    }
    P.tooWide = tooWide;
    H.haloStart.assign((size_t)nBands + 1, 0);
    for (int b = 0; b < nBands; b++) {
        H.haloStart[b + 1] = H.haloStart[b] + (int)P.halo[b].size();
        H.maxHalo = std::max(H.maxHalo, (int)P.halo[b].size());
    }
    // The check counts two vectors per tile, as when the engine could stage two: the factor is now a margin.  Changing
    // it changes the band size chosen for poorly clustered meshes.
    P.tileFits = (size_t)(bandRows + H.maxHalo + 2) * 2 * sizeof(double) <= TILE_BYTES_MAX;
    return B200LDU_OK;
}

// ---- 5. face-stream choice ------------------------------------------------------
// The face stream's CTAs hold the product buffer next to the tile.  It is used where that still leaves as many
// CTAs per SM as the entry stream's tile alone (large meshes with 512-row bands; not the one-wave bands of mid-size
// meshes nor GAMG levels with many faces per row).  B200LDU_FACE_STREAM=0 never uses it, =1 whenever it fits.
bool select_face_stream(const Plan &P)
{
    const LayoutHost &H = P.H;
    const long long tile = ((long long)H.bandRows + H.maxHalo + 1) & ~1ll;
    const bool fitsSmem = (size_t)(tile + H.fsBufMax) * sizeof(double) <= TILE_BYTES_MAX;
    if (const char *e = getenv("B200LDU_FACE_STREAM")) {
        if (!strcmp(e, "0")) return false;
        if (!strcmp(e, "1")) return P.fsFits && fitsSmem;
    }
    return P.fsFits && fitsSmem && ctas_per_sm(tile + H.fsBufMax) >= ctas_per_sm(tile);
}

// tile column of extended index t (banded row, or nPad + received slot) in band b: its own rows, then its halo list
uint16_t tile_col(const Plan &P, int b, int t)
{
    const int bandRows = P.H.bandRows, r0 = b * bandRows;
    if (t >= r0 && t < r0 + bandRows) return (uint16_t)(t - r0);
    const std::vector<int> &h = P.halo[b];
    return (uint16_t)(bandRows + (std::lower_bound(h.begin(), h.end(), t) - h.begin()));
}

// ---- 6. entry stream and the concatenated halo lists ------------------------------
void fill_entry_stream(const Graph &g, const std::vector<int> &perm, Plan &P)
{
    LayoutHost &H = P.H;
    const int bandRows = H.bandRows, slicesPerBand = bandRows / SLICE_ROWS, nPad = H.nPad;
    const std::vector<int> &iperm = P.iperm;
    std::vector<uint16_t> &col = H.col;
    std::vector<int> &code = H.code;
    col.assign((size_t)std::max<long long>(H.nEntries, 1), 0);
    code.assign(col.size(), 0);
#pragma omp parallel for schedule(dynamic, 4)
    for (int b = 0; b < H.nBands; b++) {
        const int r0 = b * bandRows;
        for (int sl = 0; sl < slicesPerBand; sl++) {
            int s = b * slicesPerBand + sl;
            long long base = H.sliceStart[s];
            int W = H.sliceW[s], WL = H.sliceWL[s];
            for (int q = 0; q < SLICE_ROWS; q++) {
                int r = s * SLICE_ROWS + q;
                int c = iperm[r];
                uint16_t self = (uint16_t)(r - r0);
                int j = 0;
                if (c >= 0) {
                    for (int f = g.ownerStart[c]; f < g.ownerStart[c + 1]; f++, j++) {
                        col[base + (long long)j * SLICE_ROWS + q] = tile_col(P, b, perm[g.u[f]]);
                        code[base + (long long)j * SLICE_ROWS + q] = 2 * f;
                    }
                    for (int k = g.losortStart[c]; k < g.losortStart[c + 1]; k++, j++) {
                        int f = g.losort[k];
                        col[base + (long long)j * SLICE_ROWS + q] = tile_col(P, b, perm[g.l[f]]);
                        code[base + (long long)j * SLICE_ROWS + q] = 2 * f + 1;
                    }
                }
                for (; j < WL; j++) { // padding: zero coefficient, own column
                    col[base + (long long)j * SLICE_ROWS + q] = self;
                    code[base + (long long)j * SLICE_ROWS + q] = -1;
                }
                if (c >= 0) {
                    for (int k = g.pfStart[c]; k < g.pfStart[c + 1]; k++, j++) {
                        col[base + (long long)j * SLICE_ROWS + q] = tile_col(P, b, nPad + g.pfItem[k]);
                        code[base + (long long)j * SLICE_ROWS + q] = -2 - g.pfItem[k];
                    }
                }
                for (; j < W; j++) {
                    col[base + (long long)j * SLICE_ROWS + q] = self;
                    code[base + (long long)j * SLICE_ROWS + q] = -1;
                }
            }
        }
    }
    H.haloIdx.assign((size_t)std::max(H.haloStart[H.nBands], 1), 0);
#pragma omp parallel for schedule(static)
    for (int b = 0; b < H.nBands; b++)
        std::copy(P.halo[b].begin(), P.halo[b].end(), H.haloIdx.begin() + H.haloStart[b]);
}

// ---- 7. face stream: owner entries, then each band's list ---------------------------
// fsCT[i]: the column and product-slot word of face-stream entry i (templates are made of them below)
void fill_face_stream(const Graph &g, const std::vector<int> &perm, Plan &P, std::vector<uint32_t> &fsCT)
{
    LayoutHost &H = P.H;
    const int bandRows = H.bandRows, slicesPerBand = bandRows / SLICE_ROWS, nPad = H.nPad;
    const std::vector<int> &iperm = P.iperm;
    // nbSlot[f]: position of face f among its neighbour cell's losort faces
    std::vector<int> nbSlot((size_t)std::max(g.nFaces, 1));
    for (int c = 0; c < g.nCells; c++)
        for (int k = g.losortStart[c]; k < g.losortStart[c + 1]; k++) nbSlot[g.losort[k]] = k - g.losortStart[c];
    std::vector<int> &fsCode = H.fsCode;
    fsCT.assign((size_t)std::max<long long>(H.fsOwn + H.fsList, 1), 0);
    fsCode.assign(fsCT.size(), 0);
    // product slot j of row n (slot 0 holds the row's owner-pass sum)
    auto slotOf = [&](int n, int j) -> uint32_t {
        const FsSlice &S = H.fsSlice[n / SLICE_ROWS];
        return (uint32_t)(S.bufOff + j * SLICE_ROWS + n % SLICE_ROWS);
    };
#pragma omp parallel for schedule(dynamic, 4)
    for (int b = 0; b < H.nBands; b++) {
        const int r0 = b * bandRows, r1 = r0 + bandRows;
        for (int sl = 0; sl < slicesPerBand; sl++) {
            const int s = b * slicesPerBand + sl;
            const FsSlice &S = H.fsSlice[s];
            const long long base = (long long)S.start64 * SLICE_ROWS;
            for (int q = 0; q < SLICE_ROWS; q++) {
                const int r = s * SLICE_ROWS + q, c = iperm[r];
                int j = 0;
                if (c >= 0) {
                    for (int f = g.ownerStart[c]; f < g.ownerStart[c + 1]; f++, j++) {
                        const int n = perm[g.u[f]];
                        const uint32_t t = (n >= r0 && n < r1) ? slotOf(n, 1 + nbSlot[f]) : FS_NONE;
                        fsCT[base + (long long)j * SLICE_ROWS + q] = tile_col(P, b, n) | t << 16;
                        fsCode[base + (long long)j * SLICE_ROWS + q] = 2 * f;
                    }
                }
                for (; j < S.wo; j++) {
                    fsCT[base + (long long)j * SLICE_ROWS + q] = (uint32_t)(r - r0) | FS_PAD << 16;
                    fsCode[base + (long long)j * SLICE_ROWS + q] = -1;
                }
            }
        }
        int ix = H.fsListStart[b], ii = H.fsListIfc[b];
        for (int r = r0; r < r1; r++) {
            const int c = iperm[r];
            if (c < 0) continue;
            for (int k = g.losortStart[c]; k < g.losortStart[c + 1]; k++) {
                const int f = g.losort[k], o = perm[g.l[f]];
                if (o >= r0 && o < r1) continue;
                fsCT[ix] = tile_col(P, b, o) | slotOf(r, 1 + (k - g.losortStart[c])) << 16;
                fsCode[ix++] = 2 * f + 1;
            }
            const int wn = H.fsSlice[r / SLICE_ROWS].wn;
            for (int k = g.pfStart[c]; k < g.pfStart[c + 1]; k++) {
                fsCT[ii] = tile_col(P, b, nPad + g.pfItem[k]) | slotOf(r, 1 + wn + (k - g.pfStart[c])) << 16;
                fsCode[ii++] = -2 - g.pfItem[k];
            }
        }
    }
}

// ---- 8. face-stream templates ---------------------------------------------------------
// The words depend on the mesh topology and the layout, not on the matrix, and on a structured mesh the slices and
// bands of the interior repeat (256^3 in 512-row bands: 163 distinct slices of 262144, 16 distinct band lists of
// 32768).  Every slice's owner block (wo x 64 words) and every band's list block becomes a reference into one table
// of distinct blocks, so that a sweep streams only the coefficients from HBM and reads the words from a table that
// stays in L2 and L1.  Owner blocks come first, so their offsets are multiples of 64; a new block is appended in
// slice order, then band order, whatever the number of threads that hashed them.
void build_face_templates(const std::vector<uint32_t> &fsCT, LayoutHost &H)
{
    const int nSlices = (int)H.fsSlice.size(), nBlocks = nSlices + H.nBands;
    auto block = [&](int k, long long &begin, long long &n) {
        if (k < nSlices) {
            begin = (long long)H.fsSlice[k].start64 * SLICE_ROWS;
            n = (long long)H.fsSlice[k].wo * SLICE_ROWS;
        } else {
            begin = H.fsListStart[k - nSlices];
            n = H.fsListStart[k - nSlices + 1] - begin;
        }
    };
    std::vector<uint64_t> hash(nBlocks);
#pragma omp parallel for schedule(dynamic, 64)
    for (int k = 0; k < nBlocks; k++) {
        long long begin, n;
        block(k, begin, n);
        uint64_t h = 0x9e3779b97f4a7c15ull ^ (uint64_t)n;
        for (long long i = 0; i < n; i++) {
            h = (h ^ fsCT[begin + i]) * 0xff51afd7ed558ccdull;
            h ^= h >> 29;
        }
        hash[k] = h;
    }
    std::unordered_map<uint64_t, std::vector<std::pair<long long, long long>>> seen; // hash -> (offset, words)
    std::vector<uint32_t> &tpl = H.fsTpl;
    tpl.clear();
    H.fsTplCount = 0;
    H.fsListTpl.assign(H.nBands, 0);
    for (int k = 0; k < nBlocks; k++) {
        long long begin, n, off = -1;
        block(k, begin, n);
        std::vector<std::pair<long long, long long>> &cand = seen[hash[k]];
        for (const auto &t : cand)
            if (t.second == n && std::equal(fsCT.begin() + begin, fsCT.begin() + begin + n, tpl.begin() + t.first)) {
                off = t.first;
                break;
            }
        if (off < 0) {
            off = (long long)tpl.size();
            tpl.insert(tpl.end(), fsCT.begin() + begin, fsCT.begin() + begin + n);
            cand.emplace_back(off, n);
            H.fsTplCount++;
        }
        if (k < nSlices)
            H.fsSlice[k].tpl64 = (int)(off / SLICE_ROWS);
        else
            H.fsListTpl[k - nSlices] = (int)off;
    }
}

// every face-stream entry's word, expanded from the templates: what the table stands for
std::vector<uint32_t> face_words(const LayoutHost &H)
{
    std::vector<uint32_t> ct((size_t)(H.fsOwn + H.fsList));
    for (const FsSlice &S : H.fsSlice)
        std::copy_n(H.fsTpl.begin() + (long long)S.tpl64 * SLICE_ROWS, (long long)S.wo * SLICE_ROWS,
                    ct.begin() + (long long)S.start64 * SLICE_ROWS);
    for (int b = 0; b < H.nBands; b++)
        std::copy_n(H.fsTpl.begin() + H.fsListTpl[b], H.fsListStart[b + 1] - H.fsListStart[b],
                    ct.begin() + H.fsListStart[b]);
    return ct;
}

// ---- 9. device path: upload the record into fixed arrays of the addressing, set every layout field of it ----
int layout_upload(b200ldu_addr *a, const Graph &g, const LayoutHost &H)
{
    LayoutDev &L = a->L;
    DeviceMem &mem = a->mem;
    TRY(mem.upload(L.sliceStart, H.sliceStart));
    TRY(mem.upload(L.sliceW, H.sliceW));
    TRY(mem.upload(L.sliceWL, H.sliceWL));
    TRY(mem.upload(L.col, H.col));
    TRY(mem.upload(a->d_code, H.code));
    TRY(mem.upload(L.haloStart, H.haloStart));
    TRY(mem.upload(L.haloIdx, H.haloIdx));
    TRY(mem.upload(L.perm, a->perm_h));
    TRY(mem.upload(L.iperm, a->iperm_h));
    TRY(mem.upload(L.sendRows, H.sendRows));
    TRY(mem.upload(a->d_l, a->l));
    TRY(mem.upload(a->d_u, a->u));
    TRY(mem.upload(a->d_ownerStart, g.ownerStart));
    TRY(mem.upload(a->d_losort, g.losort));
    TRY(mem.upload(a->d_losortStart, g.losortStart));
    if (H.nRecv) {
        TRY(mem.upload(a->d_cCellStart, g.pfStart));
        TRY(mem.upload(a->d_cCellFaces, g.pfItem));
        TRY(mem.upload(a->d_cFaceCells, a->faceCells));
    }
    if (H.hasFs) {
        TRY(mem.upload(L.fsSlice, H.fsSlice));
        TRY(mem.upload(L.fsTpl, H.fsTpl));
        TRY(mem.upload(L.fsListTpl, H.fsListTpl));
        TRY(mem.upload(a->d_fsCode, H.fsCode));
        TRY(mem.upload(L.fsListStart, H.fsListStart));
        TRY(mem.upload(L.fsListIfc, H.fsListIfc));
    }
    L.nCells = g.nCells;
    L.nPad = H.nPad;
    L.nBands = H.nBands;
    L.bandRows = H.bandRows;
    L.slicesPerBand = H.bandRows / SLICE_ROWS;
    L.nRecv = H.nRecv;
    L.maxHalo = H.maxHalo;
    L.fsBufMax = H.hasFs ? (int)H.fsBufMax : 0;
    a->nEntries = H.nEntries;
    a->nHaloTotal = H.haloStart[H.nBands];
    a->vecLen = ((long long)H.nPad + H.nRecv + 1) & ~1ll;
    a->hasFs = H.hasFs;
    a->fsOwn = H.fsOwn;
    a->fsList = H.fsList;
    a->fsTplWords = (long long)H.fsTpl.size();
    a->fsTplCount = H.fsTplCount;
    return B200LDU_OK;
}

} // namespace

int layout_build(b200ldu_addr *a, const double *centres)
{
    Graph g{a->nCells, a->nFaces, a->nPatches ? a->patchStart[a->nPatches] : 0, a->l, a->u};
    TRY(build_csr(g));
    const std::vector<int> order = renumber(g, centres);
    a->perm_h.assign(g.nCells, 0);
    for (int r = 0; r < g.nCells; r++) a->perm_h[order[r]] = r;
    csr_from_map(a->faceCells, g.nCells, g.pfStart, g.pfItem);

    int packCtas = 0;
    for (int p = 0; p < a->nPatches; p++)
        if (p < (int)a->neighbRank.size() && a->neighbRank[p] >= 0) packCtas += (a->patchStart[p + 1] - a->patchStart[p] + PACK_CHUNK - 1) / PACK_CHUNK;
    Plan P;
    for (int bandRows = pick_band_rows(g.nCells, a->ctx ? a->ctx->smCount : 132, packCtas);; bandRows /= 2) {
        TRY(plan_layout(g, order, a->perm_h, bandRows, P));
        if (!P.tooWide && P.tileFits) break;
        // poorly clustered numbering (no cell centres, high-degree graph): narrower bands shrink both the halo and the
        // tile; the row order is unchanged
        if (bandRows > SLICE_ROWS) continue;
        if (P.tooWide)
            b200_set_error("layout_build: %d band(s) of %d rows reference more than 65535 distinct columns",
                           P.tooWide, bandRows);
        else
            b200_set_error("layout_build: a band of %d rows references %d outside columns: the tile does not fit in "
                           "shared memory; pass cell centres (or renumber the mesh) so that neighbours are close",
                           bandRows, P.H.maxHalo);
        return B200LDU_ELAYOUT;
    }
    LayoutHost &H = P.H;
    H.hasFs = select_face_stream(P);
    fill_entry_stream(g, a->perm_h, P);
    // a host-only layout keeps the face stream whether or not the engine would use it, so that its structure can be checked
    if (P.fsFits && (H.hasFs || a->hostOnly)) {
        std::vector<uint32_t> fsCT;
        fill_face_stream(g, a->perm_h, P, fsCT);
        build_face_templates(fsCT, H);
    } else { // the record holds a face stream only where it was built
        H.fsSlice.clear();
        H.fsListStart.clear();
        H.fsListIfc.clear();
    }
    H.sendRows.assign(std::max(g.nRecv, 1), 0);
    for (int i = 0; i < g.nRecv; i++) H.sendRows[i] = a->perm_h[a->faceCells[i]];
    a->iperm_h.swap(P.iperm);
    if (a->hostOnly) { // structural self-check path (tests): keep the host record, no GPU
        a->host = std::move(H);
        return B200LDU_OK;
    }
    return layout_upload(a, g, H);
}

// ---------------------------------------------------------------------------
// structural self-check entry points (host only; used by the CPU test-suite to verify
// the renumbering and the banded entries without a GPU -- no arithmetic happens here)
// ---------------------------------------------------------------------------
extern "C" int b200ldu_layout_debug_create(int nCells, int nFaces, const int *lower_h, const int *upper_h,
                                           int nPatches, const int *patchStart_h, const int *faceCells_h,
                                           const double *cellCentres_h, b200ldu_addr **out)
{
    if (!out || nCells <= 0) return B200LDU_EINVAL;
    b200ldu_addr *a = new b200ldu_addr(nullptr);
    a->hostOnly = true;
    a->nCells = nCells;
    a->nFaces = nFaces;
    a->l.assign(lower_h, lower_h + nFaces);
    a->u.assign(upper_h, upper_h + nFaces);
    a->nPatches = nPatches;
    if (nPatches) {
        a->patchStart.assign(patchStart_h, patchStart_h + nPatches + 1);
        a->faceCells.assign(faceCells_h, faceCells_h + a->patchStart[nPatches]);
    }
    int rc = layout_build(a, cellCentres_h);
    if (rc != B200LDU_OK) {
        delete a;
        return rc;
    }
    *out = a;
    return B200LDU_OK;
}

// what: 0 perm(int32) 1 iperm(int32) 2 sliceStart(int64) 3 sliceW(u16) 4 sliceWL(u16) 5 col(u16)
//       6 code(int32) 7 haloStart(int32) 8 haloIdx(int32) 9 dims {nPad,nBands,bandRows,nRecv,maxHalo}(int32)
//       face stream (empty when it was not built): 10 fsSlice (4 int32 per slice: start64, bufOff, wo | wn << 16,
//       wi) 11 column and product-slot word of every entry, expanded from the templates (u32) 12 fsCode(int32)
//       13 fsListStart(int32) 14 fsListIfc(int32) 15 fs dims {fsOwn, fsList, fsBufMax, hasFs}(int64)
//       16 template table fsTpl(u32) 17 tpl64 of every slice(int32) 18 fsListTpl(int32)
// returns the element count (copies min(count, cap) elements when out != NULL)
extern "C" long long b200ldu_layout_debug_get(const b200ldu_addr *a, int what, void *out, long long cap)
{
    if (!a || !a->hostOnly) return -1;
    const LayoutHost &H = a->host;
    auto give = [&](const void *src, size_t elem, long long n) -> long long {
        if (out) memcpy(out, src, elem * (size_t)std::min(n, cap));
        return n;
    };
    const long long nFs = H.fsSlice.empty() ? 0 : H.fsOwn + H.fsList;
    int dims[5] = {H.nPad, H.nBands, H.bandRows, H.nRecv, H.maxHalo};
    std::vector<int> perSlice;
    switch (what) {
    case 0: return give(a->perm_h.data(), 4, (long long)a->perm_h.size());
    case 1: return give(a->iperm_h.data(), 4, (long long)a->iperm_h.size());
    case 2: return give(H.sliceStart.data(), 8, (long long)H.sliceStart.size());
    case 3: return give(H.sliceW.data(), 2, (long long)H.sliceW.size());
    case 4: return give(H.sliceWL.data(), 2, (long long)H.sliceWL.size());
    case 5: return give(H.col.data(), 2, H.nEntries);
    case 6: return give(H.code.data(), 4, H.nEntries);
    case 7: return give(H.haloStart.data(), 4, (long long)H.haloStart.size());
    case 8: return give(H.haloIdx.data(), 4, H.haloStart[H.nBands]);
    case 9: return give(dims, 4, 5);
    case 10:
        for (const FsSlice &S : H.fsSlice)
            perSlice.insert(perSlice.end(), {S.start64, (int)S.bufOff, S.wo | S.wn << 16, (int)S.wi});
        return give(perSlice.data(), 4, (long long)perSlice.size());
    case 11: {
        const std::vector<uint32_t> ct = nFs ? face_words(H) : std::vector<uint32_t>();
        return give(ct.data(), 4, nFs);
    }
    case 12: return give(H.fsCode.data(), 4, nFs);
    case 13: return give(H.fsListStart.data(), 4, (long long)H.fsListStart.size());
    case 14: return give(H.fsListIfc.data(), 4, (long long)H.fsListIfc.size());
    case 15: {
        long long fd[4] = {H.fsOwn, H.fsList, (int)H.fsBufMax, H.hasFs ? 1 : 0};
        return give(fd, 8, 4);
    }
    case 16: return give(H.fsTpl.data(), 4, (long long)H.fsTpl.size());
    case 17:
        for (const FsSlice &S : H.fsSlice) perSlice.push_back(S.tpl64);
        return give(perSlice.data(), 4, (long long)perSlice.size());
    case 18: return give(H.fsListTpl.data(), 4, (long long)H.fsListTpl.size());
    }
    return -1;
}

extern "C" int b200ldu_layout_debug_destroy(b200ldu_addr *a)
{
    if (a && a->hostOnly) delete a;
    return B200LDU_OK;
}
