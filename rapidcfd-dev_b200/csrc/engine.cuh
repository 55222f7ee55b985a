// engine.cuh -- the banded row-gather kernel engine (sm_90a).
//
// One CTA per band.  Phase 1 stages the band's input vector(s) into shared memory:
// the band's own rows with coalesced 128-bit loads, then the band's halo columns
// (rows of neighbouring bands or values received from coupled patches) with a sorted
// gather.  Phase 2: each warp walks its slices of 64 rows; lane k owns rows 2k, 2k+1 and
// reads slot j of both rows with one 128-bit coefficient load (double2) and one 32-bit
// column load (ushort2); the gathers hit shared memory only.  Row sums follow the
// reference's order exactly (diag, owner faces, neighbour faces, interface faces; products
// rounded separately: __dmul_rn/__dadd_rn) so results are bit-comparable with the oracle.
// Fused reductions (dot products needed by the Krylov solvers) are reduced with warp
// shuffles, then across the CTA through shared memory, and written as one partial per
// band -- summed in fixed order by the scalar-step kernel (deterministic, no atomics).
//
// Replaces the reference's Thrust functors: matrixMultiplyFunctor
// (LDU/lduMatrix/lduMatrixATmul.C:42-138), lduAddressingFunctor family
// (LDU/lduAddressing/lduAddressingFunctors.H:10-185), AINVPreconditionerFunctor
// (LDU/preconditioners/AINVPreconditioner/AINVPreconditionerF.H:5-100),
// JacobiSmootherFunctor (LDU/smoothers/Jacobi/JacobiSmootherF.H:8-110).
#pragma once
#include "internal.h"

__device__ __forceinline__ double2 ldg_stream2(const double *p)
{
    // coefficients and columns are read exactly once per kernel: keep them out of L1
    double2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];"
                 : "=d"(r.x), "=d"(r.y)
                 : "l"(p));
    return r;
}

__device__ __forceinline__ uint32_t ldg_stream_u32(const void *p)
{
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}

__device__ __forceinline__ void prefetch_l2(const void *p)
{
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

__device__ __forceinline__ void cp_async16(void *smemDst, const void *gsrc)
{
    unsigned d = (unsigned)__cvta_generic_to_shared(smemDst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}

__device__ __forceinline__ bool spin_until(const unsigned long long *f, unsigned long long seq, unsigned long long *err)
{
    // bounded wait on a flag written by a peer GPU (ld.acquire.sys): a peer that died or never entered the
    // matching kernel must not hang this GPU for ever -- after ~20 s the error word is set and the wait ends
    unsigned long long v, t0 = 0;
    unsigned spins = 0;
    for (;;) {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(f) : "memory");
        if (v >= seq) return true;
        if ((++spins & 0x3ffu) == 0) {
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (!t0) t0 = now;
            if (now - t0 > 20000000000ull) {
                if (err) atomicExch(err, 1ull);
                return false;
            }
        }
    }
}

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide sums of NRED per-thread values -> out[blockIdx.x * NRED + k].
// Fixed combination order: lanes by xor-butterfly, warps in index order.
template <int NRED, int THREADS>
__device__ __forceinline__ void block_reduce_store(double (&red)[NRED], double *partials,
                                                   int slot)
{
    __shared__ double wsum[NRED][THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NRED; k++) {
        double v = warp_sum(red[k]);
        if (lane == 0) wsum[k][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x < NRED) {
        double s = 0;
#pragma unroll
        for (int w = 0; w < THREADS / 32; w++) s += wsum[threadIdx.x][w];
        partials[(size_t)slot * NRED + threadIdx.x] = s;
    }
}

// ---------------------------------------------------------------------------
// Op concept
//   static constexpr bool STAGED true: one vector is staged in shared memory (a = its value)
//   static constexpr int  NRED   number of fused reductions (0..3)
//   static constexpr bool LOCAL  true: owner/neighbour entries only (no interfaces)
//   const int *stop              device flag; kernel exits at once when *stop != 0
//   int waitHalo                 1: a peer-memory halo exchange of the staged vector is in flight
//   bool prologue(L)             runs first in every CTA (default: nothing); false => the CTA exits
//   double *partials             [nBands*NRED]
//   double  stage(int g)         staged value at extended index g; also what the fused halo
//                                send stores for a processor-patch face cell
//   double2 stage_own(int r)     rows r, r+1 of the own band (may also write a fused vector update)
//   double  init(int r, double a)                 start of the row sum
//   double  prod(double v, double a)              the term of coefficient v and staged value a (default v*a)
//   double  add(double acc, double p)             adds a term to the row sum (default acc + p)
//   double  identity()                            p with add(acc, p) == acc bit for bit (default -0.0)
//   void    finish(int r, double acc0, double acc1, double a0, double a1, double *red)
//                                writes rows r, r+1; adds reductions
//
// Face stream (FS, symmetric matrices; layout.cu): the band's product buffer follows the tile in shared memory and
// starts filled with identity().  Pass 1 streams the owner slots of each row (the coefficients from HBM, their column and
// product-slot words from the layout's template table, which stays in L1 and L2): add(init, owner terms) in face order,
// stored in the row's slot 0, while every owner entry whose neighbour row lies in the band stores prod(v, a_own) in
// that row's neighbour slot; the CTA then stores the products of the band's list (faces owned in other bands,
// coupled-patch faces).  After one barrier pass 2 adds each row's slots in order -- neighbour faces in losort order,
// then interface faces -- so every row sum is the entry stream's, operation for operation.
// ---------------------------------------------------------------------------

// Fused halo send (peer-memory path): only operators that stage a vector and read interface
// entries ever exchange a halo, so the send is compiled for those alone.
template <class Op>
__host__ __device__ __forceinline__ bool fused_pack(const Op &op, const LayoutDev &L)
{
    return Op::STAGED && !Op::LOCAL && op.waitHalo && L.nPackChunks > 0;
}

// Predicated loads for the face stream's owner slots: when `pred` is false nothing is read (the address may lie past the
// stream) and the result is zero.  Setting the result before the predicated load ends its live range there, so a
// partial group neither keeps the previous group's registers alive nor needs a branch around its loads.
__device__ __forceinline__ double2 ldg_stream2_if(bool pred, const double *p)
{
    double2 r;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\tmov.b64 %0, 0;\n\tmov.b64 %1, 0;\n\t"
                 "@p ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%3];\n\t}"
                 : "=d"(r.x), "=d"(r.y)
                 : "r"((int)pred), "l"(p));
    return r;
}

// the face stream's words come from a small table that many slices share: keep them in L1
__device__ __forceinline__ uint2 ldg_table_u64_if(bool pred, const void *p)
{
    uint2 r;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\tmov.b32 %0, 0;\n\tmov.b32 %1, 0;\n\t"
                 "@p ld.global.nc.v2.u32 {%0, %1}, [%3];\n\t}"
                 : "=r"(r.x), "=r"(r.y)
                 : "r"((int)pred), "l"(p));
    return r;
}

// one owner entry of the face stream: ct = column | product slot << 16
template <class Op>
__device__ __forceinline__ double fs_owner(const Op &op, const double *xs, double *buf, double acc, double v,
                                           uint32_t ct, double aOwn)
{
    const uint32_t c = ct & 0xffffu, t = ct >> 16;
    if (t != FS_PAD) acc = op.add(acc, op.prod(v, Op::STAGED ? xs[c] : 0));
    if (t < FS_PAD) buf[t] = op.prod(v, aOwn);
    return acc;
}

// Owner slots per load group of the face stream's pass 1.  A hex mesh stores 3 owner faces per row, so one group covers
// nearly every slice; a group of 4 would need registers that __launch_bounds__(256, 6) leaves only by spilling.
constexpr int FS_GROUP = 3;

// Halo columns per thread taken in one load group by the staging phase: every index load of the group is issued, then
// every gather, then the shared-memory stores.  A 512-row band of a hex mesh has about 400 halo columns, so one group of 2
// covers it; the rest, if any, follow one column at a time.
constexpr int HALO_GROUP = 2;

template <class Op, bool FS>
__global__ void __launch_bounds__(ENGINE_THREADS, 6) engine_kernel(const LayoutDev L, const double *__restrict__ val, Op op)
{
    extern __shared__ double xs[];
    // Fused halo send: the first nPackChunks CTAs of the grid gather the staged vector
    // at the processor-patch face cells, store it straight into the neighbours' receive
    // buffers over NVLink and release their arrival flags; all other CTAs are SpMV bands
    // (those that reference received values wait for the neighbours' flags below).
    const bool fusedPack = fused_pack(op, L);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    // Layout words that the staging phase and pass 1 read first are streamed once per sweep, so they come from HBM.
    // None of them depends on the scalars that the prologue waits for: prefetching them into L2 now, while the prologue
    // waits, takes their round trips off the chain the band waits on, without holding a register across it.  The face
    // stream's slice descriptors and list header; the band's halo range and, one 128-byte line per lane, its halo indices.
    if (const int band = blockIdx.x - (fusedPack ? L.nPackChunks : 0); band >= 0) {
        if (FS) {
            if (lane == 0 && warp < L.slicesPerBand) prefetch_l2(L.fsSlice + band * L.slicesPerBand + warp);
            if (tid == 32) prefetch_l2(L.fsListStart + band);
            if (tid == 64) prefetch_l2(Op::LOCAL ? L.fsListIfc + band : L.fsListStart + band + 1);
            if (tid == 96) prefetch_l2(L.fsListTpl + band);
        }
        if (Op::STAGED && warp == 4) { // warp 0 waits on the gate, warps 0-3 prefetch the face stream's words
            const int hs = __ldg(L.haloStart + band), hn = __ldg(L.haloStart + band + 1) - hs;
            if (32 * lane < hn) prefetch_l2(L.haloIdx + hs + 32 * lane); // the first 1024 columns: a hint, not a copy
            if (lane == 0 && hn > 0 && hn <= 1024) prefetch_l2(L.haloIdx + hs + hn - 1);
        }
    }
    if (!op.prologue(L)) return; // stop flag (OpBase) or the deferred scalar step of the fused PCG (ops.cuh)
    unsigned long long haloSeqNow = 0;
    if (fusedPack) {
        haloSeqNow = L.seqs[1] + 1; // seqs[1] only advances when the whole grid has finished
        if ((int)blockIdx.x < L.nPackChunks) {
            const PackChunk c = L.packChunks[blockIdx.x];
            const PackPatch P = L.packPatches[c.patch];
            double *dst = P.dst[haloSeqNow & 1];
            for (int i = c.begin + threadIdx.x; i < c.end; i += ENGINE_THREADS)
                dst[i - P.start] = op.stage(__ldg(L.sendRows + i));
            __threadfence_system();
            __syncthreads();
            if (threadIdx.x == 0) {
                unsigned long long done = atomicAdd(&L.seqs[8 + c.patch], 1ull) + 1;
                if (done == (unsigned long long)P.nChunks) {
                    L.seqs[8 + c.patch] = 0;
                    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(P.flag), "l"(haloSeqNow) : "memory");
                }
                if (atomicAdd(&L.seqs[6], 1ull) + 1 == (unsigned long long)gridDim.x) {
                    L.seqs[6] = 0;
                    __threadfence();
                    L.seqs[1] = haloSeqNow;
                }
            }
            return;
        }
    }
    const int band = blockIdx.x - (fusedPack ? L.nPackChunks : 0);
    const int rowBase = band * L.bandRows;
    constexpr int NW = ENGINE_THREADS / 32;

    // ---- phase 1: stage the band's vector tile + halo ----
    // The own rows first (stage_own issues its loads before it stores a fused vector update), then the band's halo range
    // and its first group of indices, which the prefetch above has brought into L2, then the group's gathers, all issued
    // before any of them is used.  The halo range is loaded after the own rows: held across them, it spilled.
    double *const buf = xs + (Op::STAGED ? ((L.bandRows + L.maxHalo + 1) & ~1) : 0); // face stream: product buffer
    if (Op::STAGED) {
        for (int i = tid; i < (L.bandRows >> 1); i += ENGINE_THREADS)
            reinterpret_cast<double2 *>(xs)[i] = op.stage_own(rowBase + 2 * i);
        const int hs = __ldg(L.haloStart + band), hn = __ldg(L.haloStart + band + 1) - hs;
        // peer-memory halo: bands that reference received values wait for the neighbours'
        // arrival flags here, so interior bands overlap with the exchange
        const double *remoteTail = nullptr;
        if (op.waitHalo && L.haloFlags) {
            const unsigned long long seq = fusedPack ? haloSeqNow : *L.haloSeq;
            remoteTail = (seq & 1) ? L.tail1 : L.tail0;
            if (hn > 0 && __ldg(L.haloIdx + hs + hn - 1) >= L.nPad) {
                if (tid < L.nNbr) spin_until(L.haloFlags + L.nbr[tid], seq, L.seqs ? L.seqs + 7 : nullptr);
                __syncthreads();
            }
        }
        if (!remoteTail) {
            int g[HALO_GROUP];
            double h[HALO_GROUP];
#pragma unroll
            for (int k = 0; k < HALO_GROUP; k++)
                g[k] = tid + k * ENGINE_THREADS < hn ? __ldg(L.haloIdx + hs + tid + k * ENGINE_THREADS) : 0;
#pragma unroll
            for (int k = 0; k < HALO_GROUP; k++) h[k] = op.stage(g[k]); // row 0 past the halo: read, never stored
#pragma unroll
            for (int k = 0; k < HALO_GROUP; k++)
                if (tid + k * ENGINE_THREADS < hn) xs[L.bandRows + tid + k * ENGINE_THREADS] = h[k];
        }
        for (int i = remoteTail ? tid : tid + HALO_GROUP * ENGINE_THREADS; i < hn; i += ENGINE_THREADS) {
            const int gi = __ldg(L.haloIdx + hs + i);
            xs[L.bandRows + i] = (remoteTail && gi >= L.nPad) ? __ldcg(remoteTail + (gi - L.nPad)) : op.stage(gi);
        }
    }
    if (FS) {
        const double e = op.identity();
        for (int i = tid; i < (L.fsBufMax >> 1); i += ENGINE_THREADS) reinterpret_cast<double2 *>(buf)[i] = make_double2(e, e);
    }
    if (Op::STAGED || FS) __syncthreads();

    // ---- phase 2: row sums ----
    double red[Op::NRED > 0 ? Op::NRED : 1];
#pragma unroll
    for (int k = 0; k < (Op::NRED > 0 ? Op::NRED : 1); k++) red[k] = 0;

    if constexpr (FS) {
        // pass 1: owner slots, then the band's list
        for (int sl = warp; sl < L.slicesPerBand; sl += NW) {
            const FsSlice S = L.fsSlice[band * L.slicesPerBand + sl];
            const int lr = sl * SLICE_ROWS + 2 * lane;
            const double a0 = Op::STAGED ? xs[lr] : 0, a1 = Op::STAGED ? xs[lr + 1] : 0;
            double acc0 = op.init(rowBase + lr, a0);
            double acc1 = op.init(rowBase + lr + 1, a1);
            // 32-bit offsets of the lane's first slot, advanced slot by slot: the layout keeps the coefficient stream and
            // the template table below 2^31 entries (fsFits)
            unsigned vo = S.start64 * SLICE_ROWS + 2 * lane, co = S.tpl64 * SLICE_ROWS + 2 * lane;
            // slots in groups of FS_GROUP, the last one guarded by k < n: all loads of a group are issued before any use, so
            // a slice of 3 owner slots waits for one memory round trip, not three.  The uses follow in slot order, under
            // the same guard.  The own-row values are read again from the tile, which pass 1 does not write: keeping
            // them in registers across the group's loads would spill.
#pragma unroll 1
            for (int n = S.wo; n > 0; n -= FS_GROUP, vo += FS_GROUP * SLICE_ROWS, co += FS_GROUP * SLICE_ROWS) {
                double2 v[FS_GROUP];
                uint2 c[FS_GROUP];
#pragma unroll
                for (int k = 0; k < FS_GROUP; k++) {
                    v[k] = ldg_stream2_if(k < n, val + (vo + k * SLICE_ROWS));
                    c[k] = ldg_table_u64_if(k < n, L.fsTpl + (co + k * SLICE_ROWS));
                }
                const double2 a = Op::STAGED ? reinterpret_cast<const double2 *>(xs)[lr >> 1] : make_double2(0, 0);
#pragma unroll
                for (int k = 0; k < FS_GROUP; k++)
                    if (k < n) {
                        acc0 = fs_owner(op, xs, buf, acc0, v[k].x, c[k].x, a.x);
                        acc1 = fs_owner(op, xs, buf, acc1, v[k].y, c[k].y, a.y);
                    }
            }
            reinterpret_cast<double2 *>(buf + S.bufOff)[lane] = make_double2(acc0, acc1);
        }
        {
            const int ls = L.fsListStart[band], le = Op::LOCAL ? L.fsListIfc[band] : L.fsListStart[band + 1];
            const int tpl = L.fsListTpl[band] - ls; // list item i's word is fsTpl[tpl + i]
            for (int i = ls + tid; i < le; i += ENGINE_THREADS) {
                const double v = __ldcs(val + i);
                const uint32_t ct = __ldg(L.fsTpl + (tpl + i));
                buf[ct >> 16] = op.prod(v, Op::STAGED ? xs[ct & 0xffffu] : 0);
            }
        }
        __syncthreads();
        // pass 2: each row's sum, then its buffer slots in order
        for (int sl = warp; sl < L.slicesPerBand; sl += NW) {
            const FsSlice S = L.fsSlice[band * L.slicesPerBand + sl];
            const int lr = sl * SLICE_ROWS + 2 * lane;
            const double2 *bp = reinterpret_cast<const double2 *>(buf + S.bufOff) + lane;
            const double2 s0 = bp[0];
            double acc0 = s0.x, acc1 = s0.y;
            const int W = 1 + S.wn + (Op::LOCAL ? 0 : S.wi);
            for (int j = 1; j < W; j++) {
                const double2 p = bp[j * (SLICE_ROWS / 2)];
                acc0 = op.add(acc0, p.x);
                acc1 = op.add(acc1, p.y);
            }
            const double a0 = Op::STAGED ? xs[lr] : 0, a1 = Op::STAGED ? xs[lr + 1] : 0;
            op.finish(rowBase + lr, acc0, acc1, a0, a1, red);
        }
    } else
    for (int sl = warp; sl < L.slicesPerBand; sl += NW) {
        const int s = band * L.slicesPerBand + sl;
        const long long base = L.sliceStart[s];
        const int W = Op::LOCAL ? L.sliceWL[s] : L.sliceW[s];
        const int lr = sl * SLICE_ROWS + 2 * lane; // local row of this lane's first row
        const double a0 = Op::STAGED ? xs[lr] : 0, a1 = Op::STAGED ? xs[lr + 1] : 0;
        double acc0 = op.init(rowBase + lr, a0);
        double acc1 = op.init(rowBase + lr + 1, a1);
        const double *vp = val + base + 2 * lane;
        const uint16_t *cp = L.col + base + 2 * lane;
        int j = 0;
        // slots in groups of 4: all loads of a group are issued before any use
        for (; j + 4 <= W; j += 4) {
            double2 v[4];
            uint32_t c[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                v[k] = ldg_stream2(vp + (size_t)(j + k) * SLICE_ROWS);
                c[k] = ldg_stream_u32(cp + (size_t)(j + k) * SLICE_ROWS);
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int c0 = c[k] & 0xffffu, c1 = c[k] >> 16;
                acc0 = op.add(acc0, op.prod(v[k].x, Op::STAGED ? xs[c0] : 0));
                acc1 = op.add(acc1, op.prod(v[k].y, Op::STAGED ? xs[c1] : 0));
            }
        }
        for (; j < W; j++) {
            double2 v = ldg_stream2(vp + (size_t)j * SLICE_ROWS);
            uint32_t c = ldg_stream_u32(cp + (size_t)j * SLICE_ROWS);
            const int c0 = c & 0xffffu, c1 = c >> 16;
            acc0 = op.add(acc0, op.prod(v.x, Op::STAGED ? xs[c0] : 0));
            acc1 = op.add(acc1, op.prod(v.y, Op::STAGED ? xs[c1] : 0));
        }
        op.finish(rowBase + lr, acc0, acc1, a0, a1, red);
    }
    if (Op::NRED > 0) block_reduce_store<(Op::NRED > 0 ? Op::NRED : 1), ENGINE_THREADS>(red, op.partials, band);
    if (fusedPack && threadIdx.x == 0) {
        if (atomicAdd(&L.seqs[6], 1ull) + 1 == (unsigned long long)gridDim.x) {
            L.seqs[6] = 0;
            __threadfence();
            L.seqs[1] = haloSeqNow;
        }
    }
}

template <class Op, bool FS>
int engine_launch(b200ldu_addr *a, const double *val, const Op &op)
{
    const LayoutDev &L = a->L;
    size_t smem = sizeof(double) * ((Op::STAGED ? (size_t)((L.bandRows + L.maxHalo + 1) & ~1) : 0) + (FS ? (size_t)L.fsBufMax : 0));
    // the kernel also owns a little static shared memory (reduction scratch): opt in to large dynamic shared
    // memory well before the 48 KB default limit.  The attribute is per device and instantiation.
    static size_t configured[64] = {0};
    const int dev = a->ctx->device & 63;
    if (smem > 40 * 1024 && smem > configured[dev]) {
        CUDA_TRY(cudaFuncSetAttribute(engine_kernel<Op, FS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[dev] = smem;
    }
    int grid = L.nBands + (fused_pack(op, L) ? L.nPackChunks : 0);
    engine_kernel<Op, FS><<<grid, ENGINE_THREADS, smem, a->ctx->stream>>>(L, val, op);
    a->ctx->launches++;
    KERNEL_CHECK();
    return B200LDU_OK;
}

// matrix sweep with A's coefficients, or A^T's: a symmetric matrix streams its faces once (A == A^T)
template <class Op>
int engine_launch_m(b200ldu_matrix *m, bool transpose, const Op &op)
{
    if (m->d_fval) return engine_launch<Op, true>(m->a, m->d_fval, op);
    return engine_launch<Op, false>(m->a, transpose ? m->d_valT : m->d_val, op);
}
