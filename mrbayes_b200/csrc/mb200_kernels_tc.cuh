// mb200_kernels_tc.cuh -- what the tensor-core (wgmma) pruning path shares: operand geometry, the pre-split
// P(t) operand images, the node-parallel work queue.  The kernel itself is eval_tcp_kernel (mb200_kernels_tcp.cuh).
// It serves the state counts where a node update really is a dense contraction: 20-state amino-acid and 61-state codon
// models (CondLikeDown/Root_Gen*, _NY98*, CondLikeScaler_Gen*, Likelihood_Gen*; reference src/likelihood.c:204, 1575,
// 2152, 4010, 4939, 5764).
//
// Per node, per rate category, per child:   D[128 patterns][S] = CL_child[128][S] * P^T[S][S]
// is a chain of wgmma.mma_async (two 64-row warpgroup halves, kind tf32, FP32 accumulators in registers), NP/KP = S
// padded to the MMA granularity (61 -> 64/64, 20 -> 32/24).  FP32 accuracy is recovered with the 3xTF32 split
//     x = hi + lo,  hi = rna_tf32(x),  lo = rna_tf32(x - hi):   A*B ~= Ahi*Bhi + (Ahi*Blo + Alo*Bhi)
// (plain TF32 would cost ~2e-4 per product; the split leaves ~7e-7).
// The large term and the two small correction terms go to SEPARATE accumulators so that the
// tensor core's truncating accumulation bias is paid on KP/8 steps only, and are added in FP32 (RN)
// in the epilogue.
#pragma once
#include "mb200_device.cuh"
#include "gmma_common.cuh"

template <int S> struct TcGeom;
template <> struct TcGeom<61> { static constexpr int NP = 64, KP = 64, SP = 64; };
template <> struct TcGeom<20> { static constexpr int NP = 32, KP = 24, SP = 20; };

// floats per pre-split matrix image: ONE canonical-layout operand of 2 NP rows x KP -- rows [0, NP) hold the hi
// parts, rows [NP, 2 NP) the lo parts, so that  A x [B_hi | B_lo]^T  is a single N = 2 NP MMA chain (the pipelined
// kernel) and B_hi / B_lo alone are the same image addressed with N = NP (row offset 0 / NP)
template <int S> __host__ __device__ constexpr int tc_split_floats () { return 2 * TcGeom<S>::NP * TcGeom<S>::KP; }

// P(t) [S][S] row-major (row = ancestral state i) -> hi/lo rows of B[n = i][k = j] in canonical layout
template <int S>
__device__ __forceinline__ void tc_write_split_entry (float *img, int i, int j, float p)
{
    constexpr int NP = TcGeom<S>::NP;
    const float hi = gmma::to_tf32 (p), lo = gmma::to_tf32 (p - hi);
    img[gmma::canon_off (i, j, 2 * NP) / 4] = hi;
    img[gmma::canon_off (NP + i, j, 2 * NP) / 4] = lo;
}

// split images of matrices already present in the matrix buffer (set_transition_matrix, or a
// tiprobs launch predating the split buffer): grid = (matrices, K)
template <int S>
__global__ void tc_split_kernel (const float *__restrict__ matrices, float *__restrict__ split, const DevMat *__restrict__ upd,
                                 int first, int K)
{
    constexpr int NP = TcGeom<S>::NP, KP = TcGeom<S>::KP;
    const int m = upd ? upd[blockIdx.x].matrix : first + blockIdx.x, k = blockIdx.y;
    const float *P = matrices + ((size_t)m * K + k) * S * S;
    float *img = split + ((size_t)m * K + k) * tc_split_floats<S> ();
    for (int idx = threadIdx.x; idx < NP * KP; idx += blockDim.x)
        {
        const int i = idx / KP, j = idx % KP;
        tc_write_split_entry<S> (img, i, j, (i < S && j < S) ? P[i * S + j] : 0.0f);
        }
}

// =================================================================================================
// Node-parallel scheduling.  The nodes of a tree are only partially ordered: a node needs its two children, nothing
// else.  (node, 128-pattern tile) pairs are work items of a device-side queue, handed out level by level (height
// above the clean operands; host-computed) to a persistent grid; an item waits (acquire-polling a flag in global
// memory) for the items that produce its operands, which sit a whole level earlier in the queue and are therefore
// already running or done.  The critical path is (tree height x item latency), and a CTA overlaps the phases of
// independent items (mb200_kernels_tcp.cuh).
//   item id -> (slot o, evaluation e, tile t), slot-major; slots 0 .. nOp-1 are the nodes in level order, slot
//   nOp is the evaluation's closing item (site scalers in the caller's operation order, root integration).
//   flags[(e * numTiles + t) * flagStride + node] == seq  <=>  that node's rows of that tile are in memory.
// =================================================================================================
struct TcQueue
{
    unsigned int *counter;      // monotone ticket counter; base = value before this launch's first ticket
    unsigned int  base;
    int          *flags;
    int           flagStride;   // >= most operations of an evaluation + 1
    int           maxOps;       // most operations of any evaluation in this launch
    int           nEval;
    int          *error;        // set when a dependency never arrived (bounded wait)
    const int    *order;        // [total operations] level order, per evaluation at its opOff
};

__device__ __forceinline__ int tcq_ld_acquire (const int *p)
{
    int v;
    asm volatile ("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void tcq_st_release (int *p, int v)
{
    asm volatile ("st.release.gpu.global.s32 [%0], %1;\n" :: "l"(p), "r"(v) : "memory");
}

