// internal.h -- shared declarations of the b200ldu library (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/b200ldu.h"
#include "boundary_lists.cuh"

// ---------------------------------------------------------------------------
// error handling: nothing throws across the ABI
// ---------------------------------------------------------------------------
void b200_set_error(const char *fmt, ...);

#define CUDA_TRY(expr)                                                                   \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            b200_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,                 \
                           cudaGetErrorString(_e));                                      \
            return B200LDU_ECUDA;                                                        \
        }                                                                                \
    } while (0)

#define TRY(expr)                          \
    do {                                   \
        int _rc = (expr);                  \
        if (_rc != B200LDU_OK) return _rc; \
    } while (0)

#define KERNEL_CHECK() CUDA_TRY(cudaGetLastError())

// ---------------------------------------------------------------------------
// banded layout constants
// ---------------------------------------------------------------------------
// A "band" is BAND_ROWS consecutive rows of the renumbered matrix, processed by one
// CTA with the band's psi values staged in shared memory.  A "slice" is SLICE_ROWS
// consecutive rows handled by one warp, each lane owning two adjacent rows so that the
// coefficient stream is read with 128-bit loads (double2) and the 16-bit local column
// indices with 32-bit loads (ushort2).
constexpr int SLICE_ROWS = 64;
constexpr int ENGINE_THREADS = 256;

struct b200ldu_ctx {
    int device = 0;
    cudaStream_t stream = 0;
    cudaStream_t ownStream = 0; // created by ctx_create, destroyed with the context
    int smCount = 132; // H100 SXM; ctx_create reads the device
    long long launches = 0;
    // NCCL (comm.cu)
    void *nccl = nullptr; // ncclComm_t
    int rank = 0, nRanks = 1;
    struct PinnedArea *pinned = nullptr; // page-locked: the solvers' stop flags and scalar read-back (ops.cuh)
    // peer-memory (CUDA IPC over NVLink) collectives, see comm.cu
    bool p2p = false;
    char *region = nullptr;          // this rank's shared region
    char *peerRegion[8] = {nullptr}; // every rank's region mapped here (own included)
    unsigned long long *d_seq = nullptr; // local device counters: [0] reduction seq, [1] halo seq, [2..] scratch
    // device memory of the handles created on this context (DeviceMem): bytes held, allocations made
    long long memLive = 0, memAllocs = 0;
    // B200LDU_POISON_ALLOC, read by ctx_create: DeviceMem fills every new floating-point block that is not zeroNew with
    // byte 0xFF (a NaN per double), so that a result that depends on memory nobody wrote shows
    bool poison = false;
};

// Device memory of one handle (addressing, matrix, GAMG hierarchy): every device array the handle holds is allocated
// here and freed with the handle.  Fixed arrays live as long as the handle; numbered slots grow on demand and never
// shrink.  The contents of a slot are unspecified after it was reallocated, except that zeroNew zeroes a new
// allocation on the context's stream.  On a poisoning context (b200ldu_ctx::poison) a new floating-point block that is
// not zeroNew holds NaNs (byte 0xFF) instead; integer and flag arrays are never poisoned.
class DeviceMem {
  public:
    explicit DeviceMem(b200ldu_ctx *ctx) : ctx_(ctx) {}
    ~DeviceMem()
    {
        for (Block &b : fixed_) free_(b);
        for (Block &b : slots_) free_(b);
    }
    DeviceMem(const DeviceMem &) = delete;
    DeviceMem &operator=(const DeviceMem &) = delete;

    // fixed array of n (at least one) T
    template <class T>
    int alloc(T *&d, size_t n)
    {
        fixed_.emplace_back();
        return grow(fixed_.back(), d, n, false);
    }
    // slot k viewed through d, holding at least n (at least one) T: reallocated only when n is larger than it holds
    template <class T>
    int slot(int k, T *&d, size_t n, bool zeroNew = false)
    {
        if ((int)slots_.size() <= k) slots_.resize(k + 1);
        return grow(slots_[k], d, n, zeroNew);
    }
    // h uploaded into a new fixed array, or into slot k
    template <class Ptr, class T>
    int upload(Ptr &d, const std::vector<T> &h)
    {
        T *p = nullptr;
        TRY(alloc(p, h.size()));
        d = p;
        return copy_in(p, h);
    }
    template <class T>
    int upload(int k, T *&d, const std::vector<T> &h)
    {
        TRY(slot(k, d, h.size()));
        return copy_in(d, h);
    }
    void release(int k)
    {
        if (k < (int)slots_.size()) free_(slots_[k]);
    }

  private:
    struct Block {
        void *p = nullptr;
        size_t bytes = 0;
    };
    template <class T>
    int grow(Block &b, T *&d, size_t n, bool zeroNew)
    {
        const size_t bytes = sizeof(T) * (n ? n : 1);
        if (b.bytes < bytes) {
            free_(b);
            d = nullptr;
            CUDA_TRY(cudaMalloc(&b.p, bytes));
            b.bytes = bytes;
            ctx_->memLive += (long long)bytes;
            ctx_->memAllocs++;
            if (zeroNew) {
                CUDA_TRY(cudaMemsetAsync(b.p, 0, bytes, ctx_->stream));
            } else if (std::is_floating_point<T>::value && ctx_->poison) {
                // synchronised: an upload (copy_in) is not ordered after work on the context's stream
                CUDA_TRY(cudaMemsetAsync(b.p, 0xFF, bytes, ctx_->stream));
                CUDA_TRY(cudaStreamSynchronize(ctx_->stream));
            }
        }
        d = (T *)b.p;
        return B200LDU_OK;
    }
    void free_(Block &b)
    {
        if (b.bytes) cudaFree(b.p); // bytes is set once cudaMalloc succeeded
        ctx_->memLive -= (long long)b.bytes;
        b = Block();
    }
    template <class T>
    static int copy_in(T *d, const std::vector<T> &h)
    {
        if (h.size()) CUDA_TRY(cudaMemcpy(d, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice));
        return B200LDU_OK;
    }
    b200ldu_ctx *ctx_;
    std::vector<Block> fixed_, slots_;
};

// layout of the IPC-shared region of every rank
constexpr int P2P_MAXR = 8;
constexpr size_t P2P_MAIL_OFF = 0;        // double mail[2][P2P_MAXR][8]
constexpr size_t P2P_MAILFLAG_OFF = 2048; // u64 mailFlag[2][P2P_MAXR]
constexpr size_t P2P_HALOFLAG_OFF = 4096; // u64 haloFlag[P2P_MAXR]   (indexed by source rank)
constexpr int PACK_CHUNK = 4096; // faces per packing CTA of the fused halo send (comm.cu); layout.cu reserves their CTA slots
constexpr int P2P_GMAX = 256;             // doubles per rank in the coarsest-level gather
constexpr size_t P2P_GATHER_OFF = 8192;   // double gather[2][P2P_MAXR][P2P_GMAX]
constexpr size_t P2P_GFLAG_OFF = 8192 + 2 * P2P_MAXR * P2P_GMAX * sizeof(double); // u64 gflag[2][P2P_MAXR]
constexpr size_t P2P_RECV_OFF = 49152;    // double recv[2][P2P_RECV_CAP]
constexpr size_t P2P_RECV_CAP = 1u << 20; // doubles per parity
constexpr size_t P2P_REGION_BYTES = P2P_RECV_OFF + 2 * P2P_RECV_CAP * sizeof(double);
static_assert(P2P_GFLAG_OFF + 2 * P2P_MAXR * sizeof(unsigned long long) <= P2P_RECV_OFF, "gather area overlaps the receive buffers");

struct P2PRed { // passed by value to scalar_kernel
    int rank = 0, nRanks = 1;
    double *mail[P2P_MAXR] = {nullptr};
    unsigned long long *flag[P2P_MAXR] = {nullptr};
    unsigned long long *seq = nullptr;
};

// peer-memory halo send descriptors (comm.cu builds them, engine.cuh executes them)
struct PackPatch {
    double *dst[2];            // neighbour's receive buffer (parity 0/1) + this patch's offset there
    unsigned long long *flag;  // neighbour's arrival flag for this rank
    int start, n, nChunks;
};
struct PackChunk {
    int patch, begin, end;
};

// Face stream of a symmetric matrix (layout.cu, engine.cuh): every face is stored once, in its owner's row; the
// product for the neighbour's row goes through a per-band shared-memory buffer.  Per slice of 64 rows:
struct FsSlice {
    int start64;      // owner-stream offset of the slice's coefficients / 64
    int tpl64;        // offset of the slice's column and product-slot words in the template table / 64
    uint16_t bufOff;  // offset of the slice's product slots in the band's buffer (doubles; < FS_PAD)
    uint16_t wo;      // owner slots per row
    uint16_t wn, wi;  // buffer slots per row after slot 0 (the owner-pass sum): neighbour faces, then interface faces
};
static_assert(sizeof(FsSlice) == 16, "one 128-bit load per slice");
// 16-bit product-slot value of an owner entry: a buffer index, or one of these
constexpr uint32_t FS_PAD = 0xfffe;  // padding entry: contributes nothing
constexpr uint32_t FS_NONE = 0xffff; // the neighbour row lies in another band (its band's list carries the product)

// device view of the banded addressing, passed by value to kernels
struct LayoutDev {
    int nCells;         // real rows
    int nPad;           // rows incl. padding (multiple of bandRows)
    int nBands;
    int bandRows;       // rows per band (multiple of SLICE_ROWS)
    int slicesPerBand;
    int nRecv;          // halo tail length (values received from coupled patches)
    int maxHalo;        // max halo columns of any band (smem sizing)
    const long long *sliceStart; // [nSlices+1] entry offset of each slice (multiple of 64)
    const uint16_t *sliceW;      // slots per row in the slice, all entries
    const uint16_t *sliceWL;     // slots holding owner/neighbour entries only (no interfaces)
    const uint16_t *col;         // [nEntries] band-local column: < bandRows own band, else halo slot
    const int *haloStart;        // [nBands+1]
    const int *haloIdx;          // banded extended index: < nPad local row, else nPad + recv slot
    // face stream (null when the layout has none): coefficients [0, nOwn) are the slot-major owner stream, then the
    // per-band lists.  Each entry's word, column | product slot << 16, depends on the mesh and the layout alone and is
    // read from a table of distinct blocks: a slice's owner words at fsTpl + 64 tpl64 (slot-major, wo x 64 words), a
    // band's list words at fsTpl + fsListTpl[b]
    const FsSlice *fsSlice;      // [nSlices]
    const uint32_t *fsTpl;       // template table
    const int *fsListTpl;        // [nBands]
    const int *fsListStart;      // [nBands+1] list of band b: [fsListStart[b], fsListIfc[b]) faces whose owner row
    const int *fsListIfc;        // [nBands]   lies in another band, then coupled-patch faces up to fsListStart[b+1]
    int fsBufMax;                // product-buffer doubles of the largest band
    const int *perm;             // [nCells] caller cell -> banded row
    const int *iperm;            // [nPad]  banded row -> caller cell, -1 padding
    // peer-memory halo (null/0 when the exchange goes through NCCL into the vector's own tail)
    const unsigned long long *haloFlags; // this rank's arrival flags, indexed by source rank
    const unsigned long long *haloSeq;   // device counter of completed exchanges
    const double *tail0, *tail1;         // receive buffers by exchange parity
    int nNbr;
    int nbr[8];
    const PackChunk *packChunks;   // fused halo send: first nPackChunks CTAs of a consuming kernel
    const PackPatch *packPatches;
    const int *sendRows;           // banded row of every coupled-patch face cell
    unsigned long long *seqs;      // device counters: [1] halo sequence, [6] CTAs done, [8+p] chunks done
    int nPackChunks;
};

// Host arrays of the banded layout, as layout_build produces them: a device addressing uploads them (into L), the
// host-only structural self-check keeps them (b200ldu_layout_debug_get).
struct LayoutHost {
    int nPad = 0, nBands = 0, bandRows = 0, nRecv = 0, maxHalo = 0;
    long long nEntries = 0;
    // face stream: stored owner slots (padding included), list items, product-buffer doubles of the largest band,
    // and whether symmetric matrices use it
    long long fsOwn = 0, fsList = 0, fsBufMax = 0;
    bool hasFs = false;
    // entry stream
    std::vector<long long> sliceStart;
    std::vector<uint16_t> sliceW, sliceWL, col;
    std::vector<int> code;
    // halo
    std::vector<int> haloStart, haloIdx;
    std::vector<int> sendRows; // [nRecv] banded row of faceCells
    // face stream (empty where it was not built)
    std::vector<FsSlice> fsSlice;
    std::vector<uint32_t> fsTpl; // template table of the column and product-slot words
    int fsTplCount = 0;          // distinct blocks in it
    std::vector<int> fsListTpl, fsCode, fsListStart, fsListIfc;
};

// slots of b200ldu_addr::mem
enum AddrSlot {
    ADDR_X, ADDR_Y, ADDR_B,                              // banded vectors of the caller-order entry points (ldu.cu)
    ADDR_BFACE_CELLS, ADDR_BCELL_START, ADDR_BCELL_FACES, // boundary face lists (b200ldu_fv_boundary_set)
    // fvMatrix glue (fvmatrix.cu): cell fields of fvm_solve / fvm_residual, and the patch-face send buffer of
    // fv_patch_neighbour_field, which shares its slot with the component psi of fvm_solve
    ADDR_FVM_DIAG, ADDR_FVM_SOURCE, ADDR_FVM_CMPT_SOURCE, ADDR_FVM_CMPT_PSI,
    ADDR_MULES, // MULES limiter: six cell fields and the received limiters (mules.cu)
};

struct b200ldu_addr {
    explicit b200ldu_addr(b200ldu_ctx *c) : ctx(c), mem(c) {}
    b200ldu_ctx *ctx = nullptr;
    DeviceMem mem; // every device array below (fixed: the layout, cyclic sources, halo send and coupled-face lists)
    int nCells = 0, nFaces = 0;
    std::vector<int> l, u; // host copies (GAMG agglomeration, FV CSR build)
    int nPatches = 0;
    std::vector<int> patchStart, faceCells, neighbRank;
    // layout (host mirrors kept only where later setup steps need them)
    LayoutDev L{};
    long long nEntries = 0;
    long long nHaloTotal = 0;
    std::vector<int> perm_h, iperm_h;
    std::vector<double> centres_h; // optional cell centres (kept for GAMG coarse-level banding)
    int *d_code = nullptr; // [nEntries] value source: 2f+side | -1 pad | -2-pf interface
    // face stream: used by symmetric matrices when the layout has one (hasFs)
    bool hasFs = false;
    long long fsOwn = 0, fsList = 0; // stored owner slots (padding included), list items
    long long fsTplWords = 0;        // template table: words, distinct blocks
    int fsTplCount = 0;
    int *d_fsCode = nullptr; // [fsOwn + fsList] value source, as d_code
    bool p2pHalo = false;      // peer-store halo usable for this addressing
    double nCellsGlobal = 0;
    // caller-order CSR views for the FV face-sum kernels and faceH
    int *d_cyclicSrc = nullptr; // per coupled-patch face: banded row supplying it (cyclic partner) | -1
    int *d_l = nullptr, *d_u = nullptr, *d_ownerStart = nullptr, *d_losort = nullptr,
        *d_losortStart = nullptr;
    // boundary faces (all patches, patch order) and their per-cell lists; the lists are valid for nBFaces > 0 only
    int nBFaces = 0;
    int *d_bFaceCells = nullptr;
    int *d_bCellStart = nullptr, *d_bCellFaces = nullptr;
    // coupled patch faces (L.nRecv of them, patch order): per-cell lists and the face cells, uploaded when there are any
    int *d_cCellStart = nullptr, *d_cCellFaces = nullptr, *d_cFaceCells = nullptr;
    // host-only structural self-check (b200ldu_layout_debug_*): no GPU, no compute
    bool hostOnly = false;
    LayoutHost host;
    long long vecLen = 0; // nPad + nRecv (padded to even)
};

// slots of b200ldu_matrix::mem
enum MatSlot {
    MAT_WORK,                        // solver work vectors MAT_WORK + [0, MAT_NWORK) (Solve::vec; solvers.cu, gamg.cu)
    MAT_NWORK = 8,
    MAT_PSI = MAT_WORK + MAT_NWORK,  // banded psi / source of b200ldu_solve
    MAT_SRC,
    MAT_HOST_PSI, MAT_HOST_SRC,      // caller-order psi / source of b200ldu_solve_host
    MAT_HIST,                        // device residual history
    MAT_OWN_DIAG, MAT_OWN_UPPER, MAT_OWN_LOWER, MAT_OWN_BOU, MAT_OWN_INT, // caller-order copies (matrix_set)
    MAT_VAL, MAT_VALT, MAT_FVAL,     // coefficient streams (matrix_set)
};

struct b200ldu_matrix {
    explicit b200ldu_matrix(b200ldu_addr *addr) : a(addr), mem(addr->ctx) {}
    b200ldu_addr *a = nullptr;
    DeviceMem mem; // every device array below; the workspace slots are allocated once and reused across solves
                   // (PCGCache.H:9-58)
    bool symmetric = true;
    bool haveT = false;
    double *d_val = nullptr;  // banded coefficients for Amul   [nEntries]
    double *d_valT = nullptr; // banded coefficients for Tmul   (aliases d_val when symmetric)
    double *d_fval = nullptr; // face-stream coefficients [fsOwn + fsList]: a symmetric matrix has these instead of d_val
    double *d_diag = nullptr; // banded diagonal [nPad] (padding rows = 1)
    double *d_rD = nullptr;   // 1/diag, filled by matrix_set
    // views of the caller-order coefficients the matrix owns (copied by matrix_set) -- read by faceH, the fvMatrix
    // glue and the GAMG coarse-level assembly.  diag_ext is re-pointed at the boundary-folded diagonal for the
    // duration of fvm_solve; lower_ext aliases upper_ext when symmetric, int_ext aliases bou_ext when the caller
    // passed one array for both.
    const double *upper_ext = nullptr, *lower_ext = nullptr, *diag_ext = nullptr, *bou_ext = nullptr,
                 *int_ext = nullptr;
    double *d_partials = nullptr; // reduction partials
    void *d_scal = nullptr;       // SolverScalars
    double *d_sendBuf = nullptr;  // packed psi at coupled-patch face cells
};

// ---------------------------------------------------------------------------
// cross-file helpers
// ---------------------------------------------------------------------------
int layout_build(b200ldu_addr *a, const double *centres);

// a limited scheme's name and coefficient as the kernels take them (fieldops.cu): the fieldk::LIM_* code and
// 2/max(k, SMALL); an unknown name or a limitedLinear coefficient outside [0, 1] is B200LDU_EINVAL with the reference's message
int limiter_scheme(const char *scheme, double k, int *code, double *twoByk);

// banded vector of a's vecLen doubles in slot k of mem, zeroed when first allocated (its padding rows and receive tail
// rely on it); nullptr when the allocation fails
inline double *banded_vec(const b200ldu_addr *a, DeviceMem &mem, int k)
{
    double *d = nullptr;
    return mem.slot(k, d, (size_t)a->vecLen, true) == B200LDU_OK ? d : nullptr;
}

// kernel<<<ceil(nItems / block), block>>>(args...) on ctx's stream, counted in ctx->launches; nItems <= 0 launches
// nothing
template <class... P, class... A>
int launch(b200ldu_ctx *ctx, void (*kernel)(P...), long long nItems, int block, A... args)
{
    if (nItems <= 0) return B200LDU_OK;
    kernel<<<(unsigned)((nItems + block - 1) / block), block, 0, ctx->stream>>>(args...);
    ctx->launches++;
    KERNEL_CHECK();
    return B200LDU_OK;
}

// f(std::integral_constant<int, nComp>()) for a component count of 1 or 3 (the caller checks it)
template <class F>
int with_nc(int nComp, F f)
{
    return nComp == 1 ? f(std::integral_constant<int, 1>()) : f(std::integral_constant<int, 3>());
}

// stable counting sort: items of target t = the indices i with map[i] == t, ascending, at [start[t], start[t+1]);
// negative map entries belong to no target
inline void csr_from_map(const std::vector<int> &map, int nTargets, std::vector<int> &start, std::vector<int> &items)
{
    start.assign((size_t)nTargets + 1, 0);
    for (int v : map)
        if (v >= 0) start[v + 1]++;
    for (int t = 0; t < nTargets; t++) start[t + 1] += start[t];
    items.resize(std::max(start[nTargets], 1));
    std::vector<int> cur(start.begin(), start.end() - 1);
    for (int i = 0; i < (int)map.size(); i++)
        if (map[i] >= 0) items[cur[map[i]]++] = i;
}

// the boundary lists of a as the finite-volume kernels take them; a list with no faces has a null start
static inline fvmk::BoundaryLists boundary_lists(const b200ldu_addr *a)
{
    return {a->nBFaces ? a->d_bCellStart : nullptr, a->d_bCellFaces, a->L.nRecv ? a->d_cCellStart : nullptr,
            a->d_cCellFaces};
}
