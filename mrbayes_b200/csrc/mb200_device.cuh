// mb200_device.cuh -- device-side job format and buffer geometry shared by the kernels
// and the host runtime of the H100 tree-likelihood engine.
//
// Data layout in HBM (per instance == one MrBayes data division on one GPU):
//   tips      uint8  [tip][C]            (S <= 8)  state-set bitmask per pattern
//             uint64 [tip][C]            (always)  same, 64-bit
//   partials  float  [buf][k][c][Sp]     interior conditional likelihoods; Sp = S rounded
//                                        up to a multiple of 4 (61 -> 64) so that every
//                                        (k,c) row is float4-addressable / TMA-legal;
//                                        for S = 4 one (k,c) cell is exactly one float4
//   matrices  float  [mat][k][i][j]      P(t), row = ancestral state (reference layout,
//                                        src/likelihood.c:300-309)
//   scalers   float  [scaler][c]         node scalers and site scalers, one index space
//                                        like m->scalers (src/mcmc.c:6017-6046)
//   eigen     double [slot][2S + S^3]    MrBayes' cijk block (src/likelihood.c:9467)
//   weights   float  [row][c]            numSitesOfPat rows
//   invMask   uint64 [c]                 AND of all tip masks (InitInvCondLikes,
//                                        src/mcmc.c:6631-6800)
#pragma once
#include <stdint.h>

#define MB200_DEV_MAX_CATS   20
#define MB200_DEV_MAX_STATES 64

struct DevChunk                     // a run of nodes whose branches fit the shared-memory P(t) slots
                                    // (4-state path: nMat = branches | tip operands << 16 | early-fetched operands << 24)
{
    int opOff, nOp;                 // nodes    [opOff, opOff+nOp)   of the batch's operation array
    int matOff, nMat;               // branches [matOff, matOff+nMat) of the batch's chunk-matrix array
};

struct DevEval                      // one LaunchLogLikeForDivision (96 bytes)
{
    int    nMat, matOff;            // P(t) rebuilds [matOff, matOff+nMat) of the update-matrix array
                                    // (consumed by tiprobs_kernel; empty for fused batches)
    int    nOp,  opOff;             // operations     [opOff,  opOff+nOp)
    int    siteDst, siteSrc;        // -1: do not store / start from zero
    int    root, weightsRow;        // root -1: no root integration
    int    flags, hasPInvar;
    int    equalWeights;
    int    dOff;                    // doubles [dOff ...): rates[K], catW[K], freqs[S]
    double pInvar;
    int    nChunk;                  // 4-state path: chunk0 below + (nChunk-1) entries at chunkOff
    int    eigen0;                  // eigen slot of the first matrix update (normally of all of them);
                                    // -2: the evaluation carries its own cijk block after freqs in the doubles
    int    chunkOff;
    DevChunk chunk0;
    int    rootFwd;                 // 4-state path: the root buffer is the last node's result
    unsigned rootOff;               // 4-state path: float4 index of the root buffer
};
// the 4-state kernel stages a header as sizeof(DevEval)/4 words, and bench.py counts 96 bytes per evaluation
static_assert (sizeof(DevEval) == 96, "DevEval must stay 96 bytes");

// the evaluation whose matrix-update list holds update u (matOff is non-decreasing; empty lists are skipped)
__device__ __forceinline__ int owning_eval (const DevEval *evals, int nEval, int u)
{
    int e = 0;
    while (e + 1 < nEval && u >= evals[e + 1].matOff)
        e++;
    while (e > 0 && evals[e].nMat == 0)
        e--;
    return e;
}

struct DevMat                       // one branch (16 bytes)
{
    int    matrix;                  // transition-matrix buffer
    int    eigen;                   // eigen slot to rebuild P(t) from; -1 in a chunk list: clean
                                    // branch, copy the rows from the matrix buffer
    double length;
};

struct DevOp                        // one interior-node update (48 bytes)
{
    int dest, c1, m1, c2, m2, c3, m3, sw, sr;
    int s1, s2, s3;                 // fused launches: shared-memory slot of m1/m2/m3 (index into the
                                    // evaluation's matrix list, dirty first, then clean); else -1
};

// 4-state kernels: the same 48-byte record with everything address-like precomputed by pack(),
// so the node loop is  base + uniform offset  and nothing else
#define NUC_NONE     0u
#define NUC_LOAD     1u             // interior child, read from the partials buffer
#define NUC_TIP      2u             // tip child: 1-byte state mask
#define NUC_TIP_ONE  6u             // tip child under the scalar kernels' shortcut: a missing observation contributes exactly 1
#define NUC_PRE      4u             // interior child this evaluation does not write, latency path: fetched into shared
                                    // memory when the chunk starts (slot in NucOp::pad), off the node chain
#define NUC_FWD      8u             // the previous node's result: stays in registers
#define NUC_MAXPRE   8              // such operands per chunk
#define NUC_RESCALE  0x1000u
struct NucOp
{
    unsigned a1, a2, a3;            // child operand: float4 index of its partials buffer ((child - tips) * K * C)
                                    // or byte index of its tip row (child * C)
    unsigned kinds;                 // bits 0-3 / 4-7 / 8-11: kind of child 1 / 2 / 3; bit 12: rescale this node;
                                    // bits 13-18 / 19-24 / 25-30: tip-table index (within the chunk) of child 1 / 2 / 3
    unsigned destOff;               // float4 index of the destination buffer
    unsigned sp1, sp2, sp3;         // byte offset of the branch's P(t) slot in shared memory
    int sw, sr;                     // node scaler to write / to remove (-1: none)
    int dest;
    int pad;                        // bits 4j..4j+3: shared-memory slot of operand j when its kind is NUC_PRE
};
// Where the first chunk of each evaluation lives in the job blob, passed BY VALUE as a kernel
// parameter: the 4-state kernel can then issue every staging load of a CTA (evaluation header,
// branch list, node list, rates/frequencies, eigensystem) in one round instead of first fetching
// the header and then what it points to -- one memory round trip less on the latency path.
#define MB200_JOB_INDEX_MAX 16
struct JobIndexEntry { int matOff, nMat, opOff, nOp, dOff, eigen0; };     // nMat = branches | tip operands << 16
struct JobIndex
{
    int n;                          // evaluations covered (0: none, kernels read the headers first)
    int pad[3];
    JobIndexEntry e[MB200_JOB_INDEX_MAX];
};

// Resident generation kernel (mb200_replay_begin / _end): the host posts a job as 16-byte pieces in
// pinned, mapped host memory, and every piece carries the job's sequence number in .w, so a reader
// that finds the same number in every piece it read has an untorn job.
//   piece 0: count (MB200_RES_STOP: exit), blob address lo, hi     piece 1: result address lo, hi, offEval
//   piece 2: offDbl, offChunk, offCmat                             piece 3: offOp, (device copy only) done target
//   piece 4 + 2e, 5 + 2e: JobIndexEntry of evaluation e (matOff, nMat, opOff | nOp, dOff, eigen0)
#define MB200_RES_HEAD   4
#define MB200_RES_PIECES (MB200_RES_HEAD + 2 * MB200_JOB_INDEX_MAX)
#define MB200_RES_ROW    (MB200_RES_HEAD + 2)
#define MB200_RES_STOP   0x7fffffff
struct ResidentJob                  // device memory, written by the leader CTA for the others
{
    unsigned int ack;               // jobs seen, summed over the CTAs (monotone, wraps)
    unsigned int done;              // jobs finished, summed over the CTAs that ran them (monotone, wraps); a CTA adds
                                    // its 1 after its writes, so a count reached releases every write before it
    unsigned int pad[2];
    int4 row[MB200_JOB_INDEX_MAX][MB200_RES_ROW];   // per evaluation row: the job's header pieces and the row's two
                                                    // JobIndexEntry pieces, each with the sequence number in .w
};

// lanes one site pattern spreads over in the 4-state and variable-state kernels, one rate category each:
// pow2ceil(K), so that the max over a pattern's categories is an xor-shuffle
__host__ __device__ constexpr int pattern_lanes (int K)
{
    int L = 1;
    while (L < K) L <<= 1;
    return L;
}

// chunk geometry of the 4-state kernels (shared by pack() and the kernels)
__host__ __device__ constexpr int nuc_maxs (int K)          // P(t) slots per chunk
{
    return (256 / K > 96) ? 96 : 256 / K;
}
__host__ __device__ constexpr int nuc_opc (int ppb)         // nodes per chunk
{
    return (2048 / ppb > 32) ? 32 : (2048 / ppb < 8) ? 8 : 2048 / ppb;
}
// tip operands of a chunk get a 16-entry lookup table each (state mask -> P(t) column sum, per rate
// category, 256 K bytes): 96 / K tables per chunk (24 KB of shared memory), at most 64
__host__ __device__ constexpr int nuc_maxt (int K)
{
    return (96 / K > 64) ? 64 : 96 / K;
}

// Job descriptors handed over as a kernel parameter (constant bank) instead of a host->device
// copy: removes one stream operation from the latency path of small evaluations.
template <int CAP> struct alignas(16) ParamBlob { char bytes[CAP]; };
struct BlobOffsets { int eval, dbl, upd, chunk, cmat, op; };

struct DevBatchHeader
{
    int nEval, nMat, nOp, nDbl;
    // followed by DevEval[nEval], double[nDbl], DevMat upd[nMat], DevChunk[], DevMat cmat[], DevOp[nOp]
    // (each section 16-byte aligned)
};

struct DevCtx                       // instance geometry + buffer bases, passed by value
{
    int S, Sp, K, C;
    int tipCount, partialsCount, matrixCount, scalerCount, eigenCount, weightRows;
    int tilePatterns;               // patterns per CTA in the evaluation kernels
    int genKB;                      // generic kernel: rate categories whose P matrices share a pass
    int numTiles;
    int hostSum;                    // 1: every tile writes its partial lnL to the (mapped) result buffer,
                                    //    the host adds them up in tile order (small launches only)
    const uint8_t  *tip8;
    const uint64_t *tip64;
    const int      *tipPartAmbig;   // [tip] 1: some pattern is partially ambiguous (isPartAmbig)
    float          *partials;
    float          *matrices;
    float          *scalers;
    const double   *eigen;
    const float    *weights;
    const uint64_t *invMask;
    double2        *tilePartial;    // [maxEval][numTiles] per-tile lnL partial sum, and (Std) unobserved probability
    int            *tileAbort;      // [maxEval][numTiles]
    unsigned int   *ticket;         // [maxEval]
    int    cijkParts;               // eigensystems per cijk slot: 1, or K (category k uses part k: NY98-type models)
    int    patternTiles;            // 4-state path: tiles of tilePatterns patterns; numTiles (CTAs per evaluation) may be
                                    // smaller: a CTA then walks several tiles (throughput mode)
};

// ---- cross-tile lnL reduction, shared by every evaluation kernel ----
// Each tile (CTA, or tensor-core closing item) reduces its patterns' terms itself, then one thread calls
// tile_arrive; the last tile of the evaluation to arrive adds the partials (tile_sum_ltr, or a strided
// block sum above MB200_SEQ_SUM_TILES) and writes the evaluation's DevResult with dev_result_write.

// evaluations with at most this many pattern tiles add their tile partials left to right -- on the
// device (last CTA) or, on the host-call latency path, on the host: the same order, the same bits
#define MB200_SEQ_SUM_TILES 16

struct DevResult                    // 16 bytes per evaluation
{
    double lnL;
    int    status;
    int    seq;                     // launch sequence number, written LAST: a host polling the
                                    // (mapped, pinned) result sees lnL/status complete once seq matches
};

// one 16-byte store: lnL, status and the sequence number travel in a single write, so a host polling
// `seq` in (mapped, pinned) memory never sees a half-written result and no system-scope fence sits on
// the critical path.  The values are written as given (tile packets of the host-sum path included).
__device__ __forceinline__ void dev_result_write (DevResult *slot, double lnL, int status, int seq)
{
    int4 pkt;
    pkt.x = __double2loint (lnL); pkt.y = __double2hiint (lnL); pkt.z = status; pkt.w = seq;
    *reinterpret_cast<int4 *>(slot) = pkt;
}

// one thread of a tile, after the tile's reduction: publish the tile's partial and abort flag, then take
// the evaluation's ticket.  True for the last of its numTiles tiles to arrive.  (numTiles is ctx.numTiles;
// a kernel that keeps it in a register passes that, which keeps the tensor-core kernel's spills down.)
__device__ __forceinline__ bool tile_arrive (const DevCtx &ctx, int evalIdx, int numTiles, int tile, double2 partial, int abortFlag)
{
    const size_t slot = (size_t)evalIdx * numTiles + tile;
    ctx.tilePartial[slot] = partial;
    ctx.tileAbort[slot] = abortFlag;
    __threadfence ();
    return atomicAdd (&ctx.ticket[evalIdx], 1u) == (unsigned int) numTiles - 1u;
}

struct TileSum { double lnL, unobserved; int abort; };

// the last tile to arrive, one thread: the partials of every tile added left to right, abort flags OR-ed;
// then the ticket is reset for the next launch
__device__ __forceinline__ TileSum tile_sum_ltr (const DevCtx &ctx, int evalIdx, int numTiles)
{
    __threadfence ();
    TileSum r = { 0.0, 0.0, 0 };
    for (int t = 0; t < numTiles; t++)
        {
        const size_t q = (size_t)evalIdx * numTiles + t;
        r.lnL        += __ldcg (&ctx.tilePartial[q].x);
        r.unobserved += __ldcg (&ctx.tilePartial[q].y);       // dead, and not loaded, where the caller ignores it
        r.abort      |= __ldcg (&ctx.tileAbort[q]);
        }
    ctx.ticket[evalIdx] = 0u;
    return r;
}

static inline size_t mb200_align16 (size_t x) { return (x + 15) & ~(size_t)15; }
