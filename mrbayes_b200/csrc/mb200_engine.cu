// mb200_engine.cu -- host runtime + C-ABI (include/mb200.h) of the H100 tree-likelihood
// engine.  Everything a data division needs lives in HBM for the life of the instance; a
// likelihood evaluation moves a few hundred bytes of indices host->device and 12 bytes per
// chain (lnL + status) device->host.  There is no CPU fallback in this file: without an
// sm_90 device every entry point that needs the GPU fails.
#include "mb200.h"
#include "mb200_device.cuh"
#include "mb200_kernels.cuh"
#include "mb200_kernels_tc.cuh"
#include "mb200_kernels_tcp.cuh"
#include "mb200_kernels_eigen.cuh"
#include "mb200_kernels_std.cuh"

#include <cuda_runtime.h>
#include <emmintrin.h>
#include <float.h>
#include <stdio.h>
#include <time.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <memory>
#include <mutex>
#include <type_traits>
#include <utility>
#include <vector>

namespace {

// ---- resource owners: each frees what it holds when it is destroyed or assigned over, and reads as the raw
// pointer or handle it holds, which DevCtx, kernel arguments and runtime calls take as views

// a runtime call's error as an MB200 code (allocation errors are not sticky: cleared here)
int rcOf (cudaError_t e)
{
    if (e != cudaSuccess) cudaGetLastError ();
    return (e == cudaSuccess) ? MB200_SUCCESS : (e == cudaErrorMemoryAllocation) ? MB200_ERROR_OUT_OF_MEMORY : MB200_ERROR_CUDA;
}

template <class T, bool HOST>      // HOST: pinned host memory, else device memory
struct Array
{
    T *p = nullptr;
    Array () = default;
    Array (Array &&o) noexcept : p (std::exchange (o.p, nullptr)) {}
    Array &operator= (Array &&o) noexcept { std::swap (p, o.p); return *this; }
    ~Array () { if (p) { if (HOST) cudaFreeHost (p); else cudaFree (p); } }
    operator T * () const { return p; }
    int alloc (size_t n, unsigned hostFlags = cudaHostAllocDefault)    // n elements in place of the old ones, none on failure
    {
        *this = Array ();
        const int rc = rcOf (HOST ? cudaHostAlloc ((void **)&p, n * sizeof(T), hostFlags) : cudaMalloc ((void **)&p, n * sizeof(T)));
        if (rc != MB200_SUCCESS) p = nullptr;
        return rc;
    }
};
template <class T> using DevArray = Array<T, false>;
template <class T> using PinnedArray = Array<T, true>;

template <class T>
struct MappedArray : PinnedArray<T>    // pinned host memory the device reaches through `dev`
{
    T *dev = nullptr;
    int alloc (size_t n)
    {
        int rc = PinnedArray<T>::alloc (n, cudaHostAllocMapped);
        if (rc == MB200_SUCCESS) rc = rcOf (cudaHostGetDevicePointer ((void **)&dev, this->p, 0));
        if (rc != MB200_SUCCESS) *this = MappedArray ();
        return rc;
    }
};

template <class H, cudaError_t (*Destroy) (H)>
struct Handle                      // a stream or an event
{
    H h = nullptr;
    Handle () = default;
    Handle (Handle &&o) noexcept : h (std::exchange (o.h, nullptr)) {}
    ~Handle () { if (h) Destroy (h); }
    operator H () const { return h; }
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;

// n events in place of `out`'s, all created or `out` unchanged
int makeEvents (std::vector<Event> &out, int n, unsigned flags)
{
    std::vector<Event> ev (n);
    int rc = MB200_SUCCESS;
    for (int i = 0; i < n && rc == MB200_SUCCESS; i++)
        rc = rcOf (cudaEventCreateWithFlags (&ev[i].h, flags));
    if (rc == MB200_SUCCESS) out = std::move (ev);
    return rc;
}

struct Batch                       // packed evaluations (device job format)
{
    PinnedArray<char> hBlob;       // pinned host copy
    DevArray<char> dBlob;          // device copy
    size_t  cap    = 0;            // bytes allocated
    size_t  bytes  = 0;            // bytes used
    int     nEval = 0, nMat = 0, nOp = 0, nDbl = 0;
    size_t  offEval = 0, offDbl = 0, offUpd = 0, offChunk = 0, offCmat = 0, offOp = 0, offOrd = 0;
    int     maxOps = 0;            // most operations of any evaluation (tensor-core path: work-queue geometry)
    DevArray<DevResult> dRes;      // [capEval] results in HBM (device-resident replay)
    MappedArray<DevResult> hRes;   // [capEval] pinned + mapped: kernels of the host-call path write
                                   // results straight into host memory, the caller polls `seq`
    int     capEval = 0;
    int     nDirty = 0;            // P(t) rebuilds in the batch
    bool    fused = false;         // 4-state latency path: P(t) rebuilt inside the pruning kernel
    bool    needInv = false;
    bool    singleChunk = false;   // every evaluation of the batch fits one chunk (4-state path)
    int     tipEpoch = 0;          // Instance::tipEpoch at pack time (4-state records embed tip kinds)
    JobIndex jx;                   // 4-state latency path: where each evaluation's first chunk lives
    std::vector<char> hasRoot;     // [nEval] the evaluation ends in a root integration
    bool    allRoot = false;
};

struct Pending                     // the evaluation begin() started and end() has not collected yet
{
    int     count = 0;             // evaluations (0: nothing pending)
    int     seq = 0;               // sequence number the launch or post stamps into the results
    Batch  *batch = nullptr;       // whose mapped result buffer it writes
    bool    resident = false;      // posted to the resident kernel
    bool    hostSum = false;       // every tile writes its partial lnL, the host adds them up
    int     tiles = 1;             // tiles per evaluation (host sum only)
};

struct EigenSolver                     // device eigensolver staging (mb200_set_rate_matrices), built on first use
{
    size_t        inStride = 0;        // doubles per slot: [parts x S x S rate matrices | S frequencies]
    DevArray<double> dIn; PinnedArray<double> hIn;     // the staging area on the device and its pinned host copy
    MappedArray<int> status;           // non-zero = the Jacobi iteration did not converge
    DevArray<double> vec;              // [slot][part][V | V^-1], unless dFactor (which the P(t) kernel wants anyway) holds them
    DevArray<double> U;                // [slot][part][N x N] orthogonal eigenvectors of the symmetrised matrix (warm starts)
    DevArray<double2> log; DevArray<int> rounds;       // [part] rotation log and rounds of the solve in flight (stream-ordered reuse)
    std::vector<int> warmChain;        // per slot: -1 = no device eigenvectors, else warm starts since the last cold one
    std::vector<Event> evIn;           // per slot: the staging area has been read
};

struct MatRing                         // pinned ring for caller-supplied transition matrices (copied without a host wait)
{
    PinnedArray<float> buf;            // MAT_RING slots of `stride` floats
    std::vector<Event> ev;             // per slot: its copy has left the ring
    size_t        stride = 0;
    int           next = 0;            // the slot of the next call, modulo MAT_RING
};

// The kernel family that serves an instance, fixed at creation with the tile geometry in its DevCtx
enum class Family
{
    Nuc4,                              // 4 states, K <= 8: eval_nuc4_kernel and its parameter-block and resident variants
    Tensor,                            // 61-state codons (K <= 3) and 20-state amino acids (K <= 4): eval_tcp_kernel on wgmma
    Generic,                           // any other state count: eval_gen_kernel
    Std                                // variable-state (STANDARD data) divisions: eval_std_kernel
};

struct Resident                        // 4-state family: the resident generation kernel (eval_nuc4_resident_kernel)
{
    MappedArray<int4> mail;            // host -> device mailbox: MB200_RES_PIECES pieces (allocated on first use)
    DevArray<ResidentJob> job;         // the leader CTA's copy of the current job
    bool          ok = false;          // the kernel may serve this instance: its grid fits the device at once and
                                       // (once tried) its mailbox could be allocated
    bool          running = false;     // a resident kernel may still run on the stream
    double        posted = 0.0;        // host clock (s) just before the last post
};

struct TensorQueue                     // tensor-core family: pre-split P(t) images and the node-parallel work queue
{
    DevArray<float> dSplit;            // pre-split (hi, lo) canonical images of every P(t)
    DevArray<unsigned int> dCounter;   // ticket counter of the work queue (monotone)
    unsigned int  base = 0;            // its value before the next launch's first ticket
    DevArray<int> dFlags;              // [maxEval][numTiles + 1][flagStride] node-done flags (== launch sequence number)
    DevArray<int> dError;
    int           flagStride = 0;
    int           stages = 0;          // operand-ring stages of the pipelined kernel
    size_t        smem = 0;            // its dynamic shared memory
};

struct StdTables                       // variable-state family: mb200_set_pattern_states
{
    bool          ready = false;       // mb200_set_pattern_states done
    bool          uniformMk = true;    // every matrix the engine builds is an equal-frequency Mk matrix
    StdCtx        sx;
    DevArray<int> dTab;                // nStates | tiIndex | bsIndex, [3][C]
    DevArray<int2> dClasses;
    std::vector<int> hNStates, hTiIndex, hBsIndex;
    std::vector<size_t> hClOff;        // ragged host layout: offset of pattern c inside a category's block
    int           freqLen = 0;         // entries of the frequency table the patterns index: max_c (bsIndex[c] + nStates[c])
};

struct Instance
{
    Stream        stream;              // first: outlives every buffer its work may use
    mb200_instance_config cfg;
    Family        family = Family::Generic;
    DevCtx        ctx;                 // geometry and buffers; a launch changes only hostSum and throughput mode's numTiles
    DevArray<uint8_t> dTip8;
    DevArray<uint64_t> dTip64;
    DevArray<int> dTipPartAmbig;
    int           seq = 0;               // launch sequence number stamped into results
    DevArray<float> dPartials, dMatrices, dScalers, dWeights;
    DevArray<double> dEigen;
    DevArray<double> dFactor;            // large state counts: rank-one factors (U, W) of every eigensystem's c_ijk slices
    EigenSolver   eig;
    DevArray<uint64_t> dInvMask;
    DevArray<double2> dTilePartial;
    DevArray<int> dTileAbort;
    DevArray<unsigned int> dTicket;
    bool          invMaskValid = false;
    int           maxEval = 1, numSMs = 132;
    size_t        eigenStride = 0;     // doubles per eigen slot (all parts)
    int           cijkParts = 1;       // eigensystems per slot (one per category for NY98-type models)
    size_t        smemGen = 0;         // generic family: dynamic smem of eval_gen_kernel
    long long     launchKind[MB200_KERNEL_KINDS] = {0};   // per kernel family (mb200_get_kernel_launches)
    long long     launchNuc4Sub[MB200_KERNEL_COUNTERS - MB200_KERNEL_KINDS] = {0};   // 4-state sub-counts (same)
    std::vector<int> tipPartAmbig;  // host copy (operand kinds of the 4-state records)
    int           tipEpoch = 0;
    int           writtenStamp = 0;
    Pending       pending;
    Batch         scratch;             // used by the synchronous entry points
    std::vector<std::unique_ptr<Batch>> batches;   // resident batches (mb200_pack_evaluations)
    MatRing       ring;
    std::vector<int> slotOf;           // scratch: matrix index -> shared-memory slot in the current evaluation
    std::vector<int> touched;          // scratch: matrices whose slotOf entry is set
    std::vector<int> dirtyOf;          // scratch: matrix index -> index in the evaluation's update list
    std::vector<DevChunk> chunkTmp; std::vector<DevMat> cmatTmp; std::vector<int> slotTmp, nChunkTmp, tipIdxTmp, writtenTmp;
    bool          timing = false;      // bracket the evaluation kernel with events
    std::vector<Event> evA, evB;       // ring of event pairs
    long long     evCount = 0;         // pairs recorded since the last read
    Resident      res;                 // Nuc4
    TensorQueue   tc;                  // Tensor
    StdTables     vs;                  // Std
};

std::mutex               gLock;
std::vector<Instance *>  gInstances;

const int NT_GEN = 256;
const int HOSTSUM_MAX_TILES = MB200_SEQ_SUM_TILES;   // latency path: up to this many tile partials per evaluation summed on the host
const int NT_NUC4 = 256;                             // threads per CTA of the 4-state kernels
const int NT_STD = 128;                              // threads per CTA of the variable-state kernel
const int TC_MIN_ROWS = 128;                         // rows (site patterns) per tile of the tensor-core kernel = the MMA's M
const int EV_RING = 2048;

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
    fprintf (stderr, "mb200: CUDA error %s at %s:%d (%s)\n", cudaGetErrorName (e_), __FILE__, __LINE__, cudaGetErrorString (e_)); \
    return MB200_ERROR_CUDA; } } while (0)

Family familyOf (const mb200_instance_config &c)
{
    const int S = c.state_count, K = c.category_count;
    if (c.flags & MB200_CONFIG_VARIABLE_STATES) return Family::Std;
    if (S == 4 && K <= 8) return Family::Nuc4;
    if ((S == 61 && K <= 3) || (S == 20 && K <= 4)) return Family::Tensor;    // K > 1 at 61: omega categories (NY98 / M3)
    return Family::Generic;
}

// Raise `kernel`'s dynamic shared-memory limit on `device` to at least `bytes`.  The limit is one per process and
// device, and every instance there launches with it, so it only ever grows: an instance created later must not
// take away what a live one launches with.
std::map<std::pair<int, const void *>, int> gOptIn;       // (device, kernel) -> the largest limit set so far

template <class F>
cudaError_t optIn (F *kernel, int device, int bytes)
{
    std::lock_guard<std::mutex> g (gLock);
    int &have = gOptIn[{ device, (const void *) kernel }];
    if (bytes <= have) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute (kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) have = bytes;
    return e;
}

// n elements in a, zeroed on the stream
template <class A>
int zeroed (A &a, size_t n, cudaStream_t stream)
{
    const int rc = a.alloc (n);
    return rc ? rc : rcOf (cudaMemsetAsync (a, 0, n * sizeof(*a.p), stream));
}

// The 4-state kernels are compiled for K = 1..8 rate categories: calls f (std::integral_constant<int, K> ())
template <int KK = 1, class F>
int withNuc4K (int K, F &&f)
{
    if constexpr (KK > 8) return MB200_ERROR_UNSUPPORTED;
    else return (K == KK) ? f (std::integral_constant<int, KK> ()) : withNuc4K<KK + 1> (K, f);
}

// dynamic shared memory of a 4-state kernel (the parameter-block and resident kernels take the fused layout)
template <int K, bool FUSE> constexpr int nuc4Smem = (int) sizeof(Nuc4Smem<K, NT_NUC4, FUSE>);

// The tensor-core kernels are compiled for S = 20 and 61 states: calls f (std::integral_constant<int, S> ())
template <class F>
auto withTcS (int S, F &&f)
{
    return (S == 61) ? f (std::integral_constant<int, 61> ()) : f (std::integral_constant<int, 20> ());
}

// The variable-state kernel is compiled for padded state counts up to 4, 8, 12, 16 and 24: calls
// f (std::integral_constant<int, SMAX> ()) with the smallest SMAX >= Sp
template <class F>
void withStdSmax (int Sp, F &&f)
{
    if (Sp <= 4)       f (std::integral_constant<int, 4> ());
    else if (Sp <= 8)  f (std::integral_constant<int, 8> ());
    else if (Sp <= 12) f (std::integral_constant<int, 12> ());
    else if (Sp <= 16) f (std::integral_constant<int, 16> ());
    else               f (std::integral_constant<int, 24> ());
}

// dynamic shared memory of tiprobs_mm_kernel (S > 32): two S x LD double matrices
size_t mmSmem (int S)
{
    return (size_t)2 * S * ((S + 3) & ~3) * sizeof(double);
}

Instance *get (int id)
{
    std::lock_guard<std::mutex> g (gLock);
    if (id < 0 || id >= (int) gInstances.size ())
        return nullptr;
    return gInstances[id];
}

int retire (Instance *I);

// every entry point that touches the instance's stream or buffers comes through here: a resident
// kernel is stopped and waited for first
int use (Instance *I)
{
    CK (cudaSetDevice (I->cfg.device));
    return retire (I);
}

int reserveBatch (Batch &b, size_t bytes, int nEval)
{
    if (bytes > b.cap)
        {
        const size_t cap = bytes + bytes / 2 + 32768;      // never smaller than the largest parameter blob
        b.cap = 0;
        int rc = b.hBlob.alloc (cap);
        if (rc || (rc = b.dBlob.alloc (cap))) return rc;
        b.cap = cap;
        }
    if (nEval > b.capEval)
        {
        const int cap = nEval + 8;
        b.capEval = 0;
        int rc = b.dRes.alloc (cap);
        if (rc || (rc = b.hRes.alloc ((size_t) cap * HOSTSUM_MAX_TILES))) return rc;
        memset (b.hRes, 0, sizeof(DevResult) * cap * HOSTSUM_MAX_TILES);
        b.capEval = cap;
        }
    return MB200_SUCCESS;
}

bool okPartials (const Instance *I, int b, bool allowTip)
{
    return b >= (allowTip ? 0 : I->cfg.tip_count) && b < I->cfg.partials_count;
}

// ---- pack(): host evaluations -> device job format ---------------------------------------------
// One blob per batch: DevBatchHeader | DevEval[nEval] | double[nDbl] | DevMat updates[] | DevChunk[] (chunks
// after each evaluation's first) | DevMat chunk branches[] | records[nOp] | int order[nOp] (tensor-core path),
// each section 16-byte aligned.  The 4-state family's records are NucOps, every other family's DevOps.

// every count, pointer and index of the evaluations against the instance
int validate (const Instance *I, const mb200_evaluation *evs, int count)
{
    const mb200_instance_config &c = I->cfg;
    if (count < 1 || count > I->maxEval)
        return MB200_ERROR_OUT_OF_RANGE;
    const bool isStd = (I->family == Family::Std);
    if (isStd && !I->vs.ready)
        return MB200_ERROR_UNSUPPORTED;                 // mb200_set_pattern_states first
    for (int e = 0; e < count; e++)
        {
        const mb200_evaluation &ev = evs[e];
        if (ev.matrix_update_count < 0 || ev.operation_count < 0 ||
            (ev.matrix_update_count > 0 && !ev.matrix_updates) || (ev.operation_count > 0 && !ev.operations))
            return MB200_ERROR_OUT_OF_RANGE;
        if (ev.site_scaler_dst < -1 || ev.site_scaler_dst >= c.scaler_count || ev.site_scaler_src < -1 || ev.site_scaler_src >= c.scaler_count)
            return MB200_ERROR_OUT_OF_RANGE;
        if (ev.root_buffer != MB200_NONE &&
            (!okPartials (I, ev.root_buffer, false) || ev.weights_row < 0 || ev.weights_row >= c.weight_rows))
            return MB200_ERROR_OUT_OF_RANGE;
        for (int i = 0; i < ev.matrix_update_count; i++)
            {
            const mb200_matrix_update &u = ev.matrix_updates[i];
            const bool inl = (u.eigen == MB200_EIGEN_INLINE);
            if (u.matrix < 0 || u.matrix >= c.matrix_count || (!inl && !isStd && (u.eigen < 0 || u.eigen >= c.eigen_count)))
                return MB200_ERROR_OUT_OF_RANGE;
            if (inl && (!ev.inline_eigen || c.state_count != 4))
                return MB200_ERROR_UNSUPPORTED;
            if (inl != (ev.matrix_updates[0].eigen == MB200_EIGEN_INLINE))
                return MB200_ERROR_UNSUPPORTED;         // all or none of an evaluation's updates
            }
        for (int i = 0; i < ev.operation_count; i++)
            {
            const mb200_operation &op = ev.operations[i];
            if (!okPartials (I, op.dest, false) || !okPartials (I, op.child1, true) || !okPartials (I, op.child2, true) ||
                op.matrix1 < 0 || op.matrix1 >= c.matrix_count || op.matrix2 < 0 || op.matrix2 >= c.matrix_count ||
                (op.child3 != MB200_NONE && (!okPartials (I, op.child3, true) || op.matrix3 < 0 || op.matrix3 >= c.matrix_count)) ||
                op.scale_write < -1 || op.scale_write >= c.scaler_count || op.scale_remove < -1 || op.scale_remove >= c.scaler_count)
                return MB200_ERROR_OUT_OF_RANGE;
            }
        }
    return MB200_SUCCESS;
}

// 4-state family: cut an evaluation's operation list (starting at opOff of the batch) into chunks whose branches
// fit the kernel's shared-memory P(t) slots, whose nodes fit its node list and whose tip operands fit its lookup
// tables.  Appends the chunks to I->chunkTmp, their branches to I->cmatTmp and, per operation, three P(t) slots
// to I->slotTmp and three tip-table indices (-1: not a tip) to I->tipIdxTmp.  Fused: a branch the evaluation
// rebuilds carries its eigensystem and length, and dirty branches no node reads get slots too.  Returns the
// number of chunks, at least one.
int nuc4Chunks (Instance *I, const mb200_evaluation &ev, int opOff, bool fused)
{
    const mb200_instance_config &c = I->cfg;
    const int K = c.category_count;
    const int maxSlots = nuc_maxs (K), maxTips = nuc_maxt (K), opc = nuc_opc (I->ctx.tilePatterns);   // as in the kernel
    std::vector<DevChunk> &chunks = I->chunkTmp;
    std::vector<DevMat>   &cmats = I->cmatTmp;
    std::vector<int>      &touched = I->touched;        // matrices whose slotOf entry is set (the open chunk's branches)
    if ((int) I->slotOf.size () < c.matrix_count)
        { I->slotOf.assign (c.matrix_count, -1); I->dirtyOf.assign (c.matrix_count, -1); }
    for (int i = 0; i < ev.matrix_update_count; i++)
        I->dirtyOf[ev.matrix_updates[i].matrix] = i;
    DevChunk cur = { opOff, 0, (int) cmats.size (), 0 };
    int curTips = 0, n = 0;
    auto closeChunk = [&] ()
        {
        for (int m : touched) I->slotOf[m] = -1;
        touched.clear ();
        DevChunk done = cur;
        done.nMat |= curTips << 16;
        chunks.push_back (done);
        n++;
        cur.opOff += cur.nOp; cur.nOp = 0; cur.matOff = (int) cmats.size (); cur.nMat = 0; curTips = 0;
        };
    auto slotFor = [&] (int m) -> int
        {
        if (I->slotOf[m] < 0)
            {
            I->slotOf[m] = cur.nMat++;
            touched.push_back (m);
            DevMat dm; dm.matrix = m;
            int di = I->dirtyOf[m];
            if (di <= -2) di = -2 - di;       // already rebuilt in an earlier chunk: rebuild again (other
                                              // tiles must not wait for tile 0's copy in the matrix buffer)
            if (fused && di >= 0) { dm.eigen = ev.matrix_updates[di].eigen; dm.length = ev.matrix_updates[di].length; I->dirtyOf[m] = -2 - di; }
            else                  { dm.eigen = -1; dm.length = 0.0; }
            cmats.push_back (dm);
            }
        return I->slotOf[m];
        };
    for (int i = 0; i < ev.operation_count; i++)
        {
        const mb200_operation &op = ev.operations[i];
        const int m3 = (op.child3 == MB200_NONE) ? -1 : op.matrix3;
        int need = 0;
        if (I->slotOf[op.matrix1] < 0) need++;
        if (I->slotOf[op.matrix2] < 0 && op.matrix2 != op.matrix1) need++;
        if (m3 >= 0 && I->slotOf[m3] < 0 && m3 != op.matrix1 && m3 != op.matrix2) need++;
        const int tipsHere = (op.child1 < c.tip_count) + (op.child2 < c.tip_count) + (m3 >= 0 && op.child3 < c.tip_count);
        if (cur.nOp >= opc || cur.nMat + need > maxSlots || curTips + tipsHere > maxTips)
            closeChunk ();
        I->slotTmp.push_back (slotFor (op.matrix1));
        I->slotTmp.push_back (slotFor (op.matrix2));
        I->slotTmp.push_back (m3 >= 0 ? slotFor (m3) : -1);
        I->tipIdxTmp.push_back (op.child1 < c.tip_count ? curTips++ : -1);
        I->tipIdxTmp.push_back (op.child2 < c.tip_count ? curTips++ : -1);
        I->tipIdxTmp.push_back ((m3 >= 0 && op.child3 < c.tip_count) ? curTips++ : -1);
        cur.nOp++;
        }
    // fused: dirty branches no node of this evaluation reads still have to be rebuilt
    if (fused)
        for (int i = 0; i < ev.matrix_update_count; i++)
            if (I->dirtyOf[ev.matrix_updates[i].matrix] == i)
                {
                if (cur.nMat >= maxSlots) closeChunk ();
                slotFor (ev.matrix_updates[i].matrix);
                }
    if (cur.nOp > 0 || cur.nMat > 0 || n == 0)
        closeChunk ();
    for (int i = 0; i < ev.matrix_update_count; i++)
        I->dirtyOf[ev.matrix_updates[i].matrix] = -1;
    return n;
}

// 4-state family: the NucOp records of one evaluation, address-like quantities precomputed and operand kinds
// resolved.  slots / tipIdx: three per operation, from nuc4Chunks.  Also marks, per chunk, how many operands
// the latency path fetches when the chunk starts (DevChunk::nMat bits 24+), and where the root comes from.
void nuc4Encode (Instance *I, const mb200_evaluation &ev, DevEval &d, DevChunk *dc, NucOp *ops,
                 const int *slots, const int *tipIdx, bool fused)
{
    const mb200_instance_config &c = I->cfg;
    const unsigned bufStride = (unsigned) c.category_count * (unsigned) c.pattern_count;   // float4 per buffer
    const unsigned slotBytes = (unsigned) c.category_count * 80u;                           // sP[slot][K][5] float4
    const bool shortcuts = (ev.flags & MB200_FLAG_TIP_SHORTCUTS) != 0;
    auto chunk = [&] (int q) -> DevChunk & { return q == 0 ? d.chunk0 : dc[d.chunkOff + q - 1]; };
    std::vector<int> &written = I->writtenTmp;          // [buffer] == stamp: produced earlier in this evaluation
    if ((int) written.size () < c.partials_count) written.assign (c.partials_count, 0);
    const int stamp = ++I->writtenStamp;
    int prevDest = -2, q = 0, opsLeft = d.chunk0.nOp, nPre = 0;
    auto operand = [&] (int child, unsigned &a) -> unsigned
        {
        if (child == MB200_NONE) { a = 0; return NUC_NONE; }
        if (child < c.tip_count)
            {
            a = (unsigned) child * (unsigned) c.pattern_count;
            return (shortcuts && !I->tipPartAmbig[child]) ? NUC_TIP_ONE : NUC_TIP;
            }
        a = (unsigned)(child - c.tip_count) * bufStride;
        return (child == prevDest) ? NUC_FWD : NUC_LOAD;
        };
    for (int i = 0; i < ev.operation_count; i++)
        {
        const mb200_operation &op = ev.operations[i];
        NucOp &o = ops[i];
        unsigned kind[3] = { operand (op.child1, o.a1), operand (op.child2, o.a2), operand (op.child3, o.a3) };
        const int child[3] = { op.child1, op.child2, op.child3 };
        while (opsLeft == 0 && q + 1 < d.nChunk)
            {
            chunk (q++).nMat |= nPre << 24;
            opsLeft = chunk (q).nOp; nPre = 0;
            }
        // latency path: interior operands read from buffers this evaluation does not write are
        // fetched into shared memory when the chunk starts, off the node-to-node chain
        o.pad = 0;
        for (int j = 0; j < 3; j++)
            if (fused && kind[j] == NUC_LOAD && written[child[j]] != stamp && nPre < NUC_MAXPRE)
                {
                kind[j] = NUC_PRE;
                o.pad |= nPre << (4 * j);
                nPre++;
                }
        o.kinds = kind[0] | (kind[1] << 4) | (kind[2] << 8) | (op.scale_write >= 0 ? NUC_RESCALE : 0u);
        for (int j = 0; j < 3; j++)
            if (tipIdx[3*i + j] >= 0)
                o.kinds |= (unsigned) tipIdx[3*i + j] << (13 + 6 * j);
        o.destOff = (unsigned)(op.dest - c.tip_count) * bufStride;
        o.sp1 = (unsigned) slots[3*i] * slotBytes;
        o.sp2 = (unsigned) slots[3*i + 1] * slotBytes;
        o.sp3 = (slots[3*i + 2] >= 0) ? (unsigned) slots[3*i + 2] * slotBytes : 0u;
        o.sw = op.scale_write; o.sr = op.scale_remove; o.dest = op.dest;
        opsLeft--;
        prevDest = op.dest;
        written[op.dest] = stamp;
        }
    chunk (q).nMat |= nPre << 24;
    d.rootFwd = (ev.root_buffer != MB200_NONE && ev.root_buffer == prevDest) ? 1 : 0;
    d.rootOff = (ev.root_buffer != MB200_NONE) ? (unsigned)(ev.root_buffer - c.tip_count) * bufStride : 0u;
}

// tensor-core path: the nodes of an evaluation are work items of a device-side queue; an item waits for the
// items that produce its operands.  s1/s2/s3 = producing operation (index within the evaluation) or -1 (tip, or
// a buffer this evaluation does not write); the queue hands the nodes out level by level (height above the clean
// operands) so that dependent items sit far apart in it
void tcOrder (Instance *I, DevOp *ops, int nOp, int *order)
{
    const int tips = I->cfg.tip_count;
    std::vector<int> &producer = I->writtenTmp;         // [buffer] -> operation index + 1 (0: none), reset per evaluation
    if ((int) producer.size () < I->cfg.partials_count) producer.assign (I->cfg.partials_count, 0);
    std::vector<int> level (nOp, 0);
    for (int i = 0; i < nOp; i++)
        {
        DevOp &o = ops[i];
        const int ch[3] = { o.c1, o.c2, o.c3 };
        int pr[3], lv = 0;
        for (int j = 0; j < 3; j++)
            {
            pr[j] = (ch[j] >= tips && producer[ch[j]] > 0) ? producer[ch[j]] - 1 : -1;
            if (pr[j] >= 0 && level[pr[j]] + 1 > lv) lv = level[pr[j]] + 1;
            }
        o.s1 = pr[0]; o.s2 = pr[1]; o.s3 = pr[2];
        level[i] = lv;
        producer[o.dest] = i + 1;
        }
    for (int i = 0; i < nOp; i++)
        producer[ops[i].dest] = 0;
    int pos = 0;
    for (int lv = 0; pos < nOp; lv++)
        for (int i = 0; i < nOp; i++)
            if (level[i] == lv)
                order[pos++] = i;
}

// validate + flatten host evaluations into the device job format
int pack (Instance *I, Batch &b, const mb200_evaluation *evs, int count)
{
    int rc = validate (I, evs, count);
    if (rc != MB200_SUCCESS)
        return rc;
    const mb200_instance_config &c = I->cfg;
    const int K = c.category_count, S = c.state_count;
    const bool nuc4 = (I->family == Family::Nuc4), tensor = (I->family == Family::Tensor);
    // state frequencies per evaluation: S, or the whole table for variable-state divisions (one vector per state count)
    const int  nFreq = (I->family == Family::Std) ? MB200_MAX_STATES : S;
    const long tiles = I->ctx.patternTiles;
    // fused P(t) rebuild (every CTA rebuilds the dirty matrices of its evaluation): small launches (latency-
    // bound regime), and launches of many evaluations over few pattern tiles each (the rebuild is repeated
    // only tiles-per-evaluation times, and a second kernel + its launch gap would cost more)
    const bool fused = nuc4 && (tiles * count <= 4L * I->numSMs || tiles <= 16);

    std::vector<DevChunk> &chunks = I->chunkTmp;        // every evaluation's chunks, its first included
    std::vector<int>      &nChunkOf = I->nChunkTmp;
    chunks.clear (); I->cmatTmp.clear (); I->slotTmp.clear (); I->tipIdxTmp.clear (); nChunkOf.assign (count, 0);
    int nMat = 0, nOp = 0;
    for (int e = 0; e < count; e++)
        {
        if (nuc4)
            nChunkOf[e] = nuc4Chunks (I, evs[e], nOp, fused);
        nMat += evs[e].matrix_update_count;
        nOp  += evs[e].operation_count;
        }

    // ---- layout ----
    const int nUpd = fused ? 0 : nMat;                 // update list only feeds the stand-alone P(t) kernel
    const int nExtraChunks = (int) chunks.size () - (nuc4 ? count : 0);    // the first chunk lives in the DevEval
    // per evaluation: rates[K], catW[K], freqs[S] and, when the evaluation carries its own
    // eigensystem, the cijk block [2S + S^3]
    int nDbl = 0;
    for (int e = 0; e < count; e++)
        nDbl += 2*K + nFreq + (evs[e].inline_eigen ? 2*S + S*S*S : 0);
    nDbl = (nDbl + 1) & ~1;
    size_t offEval  = mb200_align16 (sizeof(DevBatchHeader));
    size_t offDbl   = mb200_align16 (offEval + sizeof(DevEval) * (size_t)count);
    size_t offUpd   = mb200_align16 (offDbl + sizeof(double) * (size_t)nDbl);
    size_t offChunk = mb200_align16 (offUpd + sizeof(DevMat) * (size_t)nUpd);
    size_t offCmat  = mb200_align16 (offChunk + sizeof(DevChunk) * (size_t)nExtraChunks);
    size_t offOp    = mb200_align16 (offCmat + sizeof(DevMat) * I->cmatTmp.size ());
    size_t offOrd   = mb200_align16 (offOp + sizeof(DevOp) * (size_t)nOp);      // tensor-core path: level order of the operations
    size_t bytes    = mb200_align16 (offOrd + (tensor ? sizeof(int) * (size_t)nOp : 0));
    rc = reserveBatch (b, bytes, count);
    if (rc != MB200_SUCCESS)
        return rc;
    DevBatchHeader *h = (DevBatchHeader *) b.hBlob.p;
    h->nEval = count; h->nMat = nUpd; h->nOp = nOp; h->nDbl = nDbl;
    DevEval  *de = (DevEval  *)(b.hBlob + offEval);
    double   *dd = (double   *)(b.hBlob + offDbl);
    DevMat   *du = (DevMat   *)(b.hBlob + offUpd);
    DevChunk *dc = (DevChunk *)(b.hBlob + offChunk);
    DevOp    *dops = (DevOp  *)(b.hBlob + offOp);
    int      *dord = (int    *)(b.hBlob + offOrd);
    if (!I->cmatTmp.empty ())
        memcpy (b.hBlob + offCmat, I->cmatTmp.data (), sizeof(DevMat) * I->cmatTmp.size ());

    // ---- per evaluation: header, doubles, updates, then the records of its kernel family ----
    b.maxOps = 0;
    b.needInv = false;
    b.jx.n = (fused && count <= MB200_JOB_INDEX_MAX) ? count : 0;
    int mOff = 0, oOff = 0, chunkPos = 0, extraPos = 0, dblPos = 0;
    for (int e = 0; e < count; e++)
        {
        const mb200_evaluation &ev = evs[e];
        DevEval &d = de[e];
        memset (&d, 0, sizeof(d));
        d.nMat = fused ? 0 : ev.matrix_update_count; d.matOff = mOff;
        d.nOp  = ev.operation_count;     d.opOff  = oOff;
        d.siteDst = ev.site_scaler_dst;  d.siteSrc = ev.site_scaler_src;
        d.root = ev.root_buffer;         d.weightsRow = ev.weights_row;
        d.flags = ev.flags;              d.hasPInvar = ev.has_p_invar ? 1 : 0;
        d.pInvar = ev.p_invar;
        d.dOff = dblPos;
        dblPos += 2*K + nFreq + (ev.inline_eigen ? 2*S + S*S*S : 0);
        d.eigen0 = (ev.matrix_update_count > 0) ? ev.matrix_updates[0].eigen : 0;
        d.nChunk = nChunkOf[e];
        d.chunkOff = extraPos;
        if (nChunkOf[e] > 0)
            {
            d.chunk0 = chunks[chunkPos];
            for (int q = 1; q < nChunkOf[e]; q++)
                dc[extraPos++] = chunks[chunkPos + q];
            chunkPos += nChunkOf[e];
            }
        if (d.root != MB200_NONE && d.hasPInvar) b.needInv = true;
        double *dv = dd + d.dOff;
        bool eq = true;
        for (int k = 0; k < K; k++)
            {
            dv[k]     = ev.category_rates[k];
            dv[K + k] = ev.category_weights[k];
            if (ev.category_weights[k] != ev.category_weights[0]) eq = false;
            }
        d.equalWeights = eq ? 1 : 0;
        for (int s = 0; s < nFreq; s++)
            dv[2*K + s] = ev.state_freqs[s];
        if (ev.inline_eigen)
            memcpy (dv + 2*K + S, ev.inline_eigen, sizeof(double) * (size_t)(2*S + S*S*S));
        if (!fused)
            for (int i = 0; i < ev.matrix_update_count; i++)
                {
                const mb200_matrix_update &u = ev.matrix_updates[i];
                DevMat &m = du[mOff + i];
                m.matrix = u.matrix; m.eigen = u.eigen; m.length = u.length;
                }
        if (nuc4)
            {
            nuc4Encode (I, ev, d, dc, reinterpret_cast<NucOp *>(dops) + oOff, I->slotTmp.data () + 3 * (size_t)oOff,
                        I->tipIdxTmp.data () + 3 * (size_t)oOff, fused);
            if (e < b.jx.n)
                b.jx.e[e] = { d.chunk0.matOff, d.chunk0.nMat, d.chunk0.opOff, d.chunk0.nOp, d.dOff, d.eigen0 };
            }
        else
            {
            for (int i = 0; i < ev.operation_count; i++)
                {
                const mb200_operation &op = ev.operations[i];
                DevOp &o = dops[oOff + i];
                o.dest = op.dest; o.c1 = op.child1; o.m1 = op.matrix1; o.c2 = op.child2; o.m2 = op.matrix2;
                o.c3 = op.child3; o.m3 = (op.child3 == MB200_NONE) ? MB200_NONE : op.matrix3;
                o.sw = op.scale_write; o.sr = op.scale_remove;
                o.s1 = o.s2 = o.s3 = -1;
                }
            if (tensor)
                {
                tcOrder (I, dops + oOff, ev.operation_count, dord + oOff);
                if (ev.operation_count > b.maxOps) b.maxOps = ev.operation_count;
                }
            }
        mOff += fused ? 0 : ev.matrix_update_count;
        oOff += ev.operation_count;
        }
    b.hasRoot.resize (count);
    b.allRoot = true;
    for (int e = 0; e < count; e++)
        {
        b.hasRoot[e] = (evs[e].root_buffer != MB200_NONE);
        if (!b.hasRoot[e]) b.allRoot = false;
        }
    b.bytes = bytes; b.nEval = count; b.nMat = nUpd; b.nOp = nOp; b.nDbl = nDbl;
    b.nDirty = nMat; b.fused = fused; b.tipEpoch = I->tipEpoch;
    b.singleChunk = true;
    for (int e = 0; e < count; e++) if (nChunkOf[e] != 1) b.singleChunk = false;
    b.offEval = offEval; b.offDbl = offDbl; b.offUpd = offUpd; b.offChunk = offChunk; b.offCmat = offCmat; b.offOp = offOp; b.offOrd = offOrd;
    return MB200_SUCCESS;
}

int ensureInvMask (Instance *I)
{
    if (I->invMaskValid)
        return MB200_SUCCESS;
    int C = I->cfg.pattern_count;
    invmask_kernel<<<(C + 255) / 256, 256, 0, I->stream>>> (I->dInvMask, I->dTip64, I->cfg.tip_count, C);
    CK (cudaGetLastError ());
    I->launchKind[MB200_KERNEL_SETUP]++;
    I->invMaskValid = true;
    return MB200_SUCCESS;
}

constexpr int PARAM_SMALL = 4096, PARAM_MID = 10240, PARAM_BIG = 30720;   // parameter-block sizes compiled (the launch copies all of it)

bool paramEligible (const Instance *I, const Batch &b)
{
    return b.fused && b.bytes <= (size_t) PARAM_BIG;
}

// make the evaluation just launched or posted the instance's pending one: runEnd () and retire () read
// only this record
void setPending (Instance *I, Batch &b, int seq, bool resident, bool hostSum, int tiles)
{
    I->pending = { b.nEval, seq, &b, resident, hostSum, tiles };
}

// ---- per-family launch: the P(t) kernel the batch needs, then the evaluation kernel ----

template <class T> const T *blobAt (const Batch &b, size_t off) { return (const T *)(b.dBlob + off); }

// P(t) of the batch's matrix updates, one CTA per (update, category): above 32 states from the rank-one factors
// (dFactor is always allocated there), writing the tensor-core family's pre-split images too when `split` is given
int tiprobs (Instance *I, const Batch &b, const DevCtx &ctx, float *split)
{
    const DevEval *de = blobAt<DevEval> (b, b.offEval);
    const double  *dd = blobAt<double> (b, b.offDbl);
    const DevMat  *du = blobAt<DevMat> (b, b.offUpd);
    const dim3 grid (b.nMat, ctx.K);
    if (ctx.S > 32)
        tiprobs_mm_kernel<<<grid, 256, mmSmem (ctx.S), I->stream>>> (ctx, de, b.nEval, dd, du, I->dFactor, split);
    else
        tiprobs_kernel<<<grid, 128, 0, I->stream>>> (ctx, de, b.nEval, dd, du);
    CK (cudaGetLastError ());
    I->launchKind[MB200_KERNEL_TIPROBS]++;
    return MB200_SUCCESS;
}

// kernel timing brackets the evaluation kernel (and the tensor family's image split), not the P(t) kernel before it
int timingStart (Instance *I)
{
    if (I->timing)
        CK (cudaEventRecord (I->evA[I->evCount % EV_RING], I->stream));
    return MB200_SUCCESS;
}

int launchNuc4 (Instance *I, const Batch &b, DevCtx &ctx, bool viaParams, bool toHost, DevResult *res, int seq)
{
    int rc = (b.nDirty > 0 && !b.fused) ? tiprobs (I, b, ctx, nullptr) : MB200_SUCCESS;
    if (!rc) rc = timingStart (I);
    if (rc) return rc;
    // throughput mode (MB200_CONFIG_THROUGHPUT): several analyses share the GPU, so SM time counts, not
    // the latency of one launch -- one CTA per evaluation walks all its tiles and builds P(t) once
    // instead of once per tile.  Single-chunk evaluations only (per-pattern state lives in registers).
    if (b.fused && (I->cfg.flags & MB200_CONFIG_THROUGHPUT) && b.singleChunk)
        {
        ctx.numTiles = 1;
        I->launchNuc4Sub[MB200_KERNEL_NUC4_PER_EVAL - MB200_KERNEL_KINDS]++;
        }
    ctx.hostSum = (toHost && b.allRoot && b.fused && ctx.numTiles <= HOSTSUM_MAX_TILES) ? 1 : 0;
    const dim3 grid (ctx.numTiles, b.nEval);
    const BlobOffsets off = { (int) b.offEval, (int) b.offDbl, (int) b.offUpd, (int) b.offChunk, (int) b.offCmat, (int) b.offOp };
    const DevEval  *de = blobAt<DevEval> (b, b.offEval);
    const double   *dd = blobAt<double> (b, b.offDbl);
    const DevChunk *dc = blobAt<DevChunk> (b, b.offChunk);
    const DevMat   *dm = blobAt<DevMat> (b, b.offCmat);
    const DevOp    *dops = blobAt<DevOp> (b, b.offOp);
    rc = withNuc4K (ctx.K, [&] (auto k)
        {
        constexpr int KK = decltype (k)::value;
        // the job descriptors in the parameter block (no H2D copy); the launch copies all CAP bytes
        auto viaBlock = [&] (auto cap)
            {
            constexpr int CAP = decltype (cap)::value;
            eval_nuc4_pkernel<KK, NT_NUC4, CAP><<<grid, NT_NUC4, nuc4Smem<KK, true>, I->stream>>> (
                ctx, off, res, seq, b.jx, *reinterpret_cast<const ParamBlob<CAP> *>(b.hBlob.p));
            };
        if (!viaParams && b.fused)
            eval_nuc4_kernel<KK, NT_NUC4, true><<<grid, NT_NUC4, nuc4Smem<KK, true>, I->stream>>> (ctx, de, dd, dc, dm, dops, res, seq, b.jx);
        else if (!viaParams)
            eval_nuc4_kernel<KK, NT_NUC4, false><<<grid, NT_NUC4, nuc4Smem<KK, false>, I->stream>>> (ctx, de, dd, dc, dm, dops, res, seq, b.jx);
        else if (b.bytes <= (size_t) PARAM_SMALL)
            viaBlock (std::integral_constant<int, PARAM_SMALL> ());
        else if (b.bytes <= (size_t) PARAM_MID)
            viaBlock (std::integral_constant<int, PARAM_MID> ());
        else
            viaBlock (std::integral_constant<int, PARAM_BIG> ());
        return MB200_SUCCESS;
        });
    if (rc != MB200_SUCCESS) return rc;
    I->launchKind[MB200_KERNEL_NUC4]++;
    if (viaParams)
        I->launchNuc4Sub[MB200_KERNEL_NUC4_PARAMS - MB200_KERNEL_KINDS]++;
    return MB200_SUCCESS;
}

int launchTensor (Instance *I, const Batch &b, const DevCtx &ctx, DevResult *res, int seq)
{
    return withTcS (ctx.S, [&] (auto s)
        {
        constexpr int TS = decltype (s)::value;
        // 61 states: tiprobs_mm_kernel writes the pre-split images of the matrices it rebuilds
        int rc = (b.nDirty > 0) ? tiprobs (I, b, ctx, (TS == 61) ? I->tc.dSplit.p : nullptr) : MB200_SUCCESS;
        if (!rc) rc = timingStart (I);
        if (rc) return rc;
        if constexpr (TS != 61)
            if (b.nDirty > 0)
                {
                tc_split_kernel<TS><<<dim3 (b.nMat, ctx.K), 128, 0, I->stream>>> (I->dMatrices, I->tc.dSplit, blobAt<DevMat> (b, b.offUpd), 0, ctx.K);
                CK (cudaGetLastError ());
                I->launchKind[MB200_KERNEL_SETUP]++;
                }
        // warp-specialised pipeline over the node-parallel queue: one persistent CTA per SM
        TcQueue Q;
        Q.counter = I->tc.dCounter; Q.base = I->tc.base; Q.flags = I->tc.dFlags; Q.flagStride = I->tc.flagStride;
        Q.maxOps = b.maxOps; Q.nEval = b.nEval; Q.error = I->tc.dError; Q.order = blobAt<int> (b, b.offOrd);
        const long total = (long)(b.maxOps + 1) * b.nEval * ctx.numTiles;
        const int  g = (int)((total < (long) I->numSMs) ? total : (long) I->numSMs);
        I->tc.base += (unsigned int)(total + g);                  // every CTA draws exactly one ticket past the end
        eval_tcp_kernel<TS><<<g, TCP_THREADS, I->tc.smem, I->stream>>> (ctx, Q, I->tc.stages, blobAt<DevEval> (b, b.offEval),
                                                                       blobAt<double> (b, b.offDbl), blobAt<DevOp> (b, b.offOp), I->tc.dSplit, res, seq);
        I->launchKind[MB200_KERNEL_TENSOR]++;
        return MB200_SUCCESS;
        });
}

int launchGeneric (Instance *I, const Batch &b, const DevCtx &ctx, DevResult *res, int seq)
{
    int rc = (b.nDirty > 0) ? tiprobs (I, b, ctx, nullptr) : MB200_SUCCESS;
    if (!rc) rc = timingStart (I);
    if (rc) return rc;
    eval_gen_kernel<NT_GEN><<<dim3 (ctx.numTiles, b.nEval), NT_GEN, I->smemGen, I->stream>>> (
        ctx, blobAt<DevEval> (b, b.offEval), blobAt<double> (b, b.offDbl), blobAt<DevOp> (b, b.offOp), res, seq);
    I->launchKind[MB200_KERNEL_GENERIC]++;
    return MB200_SUCCESS;
}

int launchStd (Instance *I, const Batch &b, const DevCtx &ctx, DevResult *res, int seq)
{
    const DevEval *de = blobAt<DevEval> (b, b.offEval);
    const double  *dd = blobAt<double> (b, b.offDbl);
    if (b.nDirty > 0)
        {
        tiprobs_std_kernel<<<b.nMat, 64, 0, I->stream>>> (ctx, I->vs.sx, de, b.nEval, dd, blobAt<DevMat> (b, b.offUpd));
        CK (cudaGetLastError ());
        I->launchKind[MB200_KERNEL_TIPROBS]++;
        }
    int rc = timingStart (I);
    if (rc) return rc;
    const DevOp *dops = blobAt<DevOp> (b, b.offOp);
    const int mk = I->vs.uniformMk ? 1 : 0;
    withStdSmax (ctx.Sp, [&] (auto smax)
        {
        eval_std_kernel<decltype (smax)::value, NT_STD><<<dim3 (ctx.numTiles, b.nEval), NT_STD, 0, I->stream>>> (
            ctx, I->vs.sx, de, dd, dops, res, seq, mk);
        });
    I->launchKind[MB200_KERNEL_STD]++;
    return MB200_SUCCESS;
}

// launch the evaluation of a packed batch.  viaParams: the job lives in b.hBlob only and rides in the
// parameter block (otherwise the caller has copied it to dBlob).  toHost: the results go to the batch's
// mapped host buffer and the launch becomes the pending evaluation; else they go to b.dRes.
int launch (Instance *I, Batch &b, bool viaParams, bool toHost)
{
    DevResult *res = toHost ? b.hRes.dev : b.dRes;
    DevCtx ctx = I->ctx;
    const int seq = ++I->seq;
    int rc = b.needInv ? ensureInvMask (I) : MB200_SUCCESS;
    if (rc != MB200_SUCCESS) return rc;
    switch (I->family)
        {
        case Family::Nuc4:    rc = launchNuc4 (I, b, ctx, viaParams, toHost, res, seq); break;
        case Family::Tensor:  rc = launchTensor (I, b, ctx, res, seq); break;
        case Family::Generic: rc = launchGeneric (I, b, ctx, res, seq); break;
        case Family::Std:     rc = launchStd (I, b, ctx, res, seq); break;
        }
    if (rc != MB200_SUCCESS) return rc;
    CK (cudaGetLastError ());
    if (I->timing)
        {
        CK (cudaEventRecord (I->evB[I->evCount % EV_RING], I->stream));
        I->evCount++;
        }
    if (toHost)
        setPending (I, b, seq, false, ctx.hostSum != 0, ctx.numTiles);
    return MB200_SUCCESS;
}

// ---- per-family setup (at creation): tile geometry into I->ctx, the dynamic shared memory of the kernels the
// family launches, family-only buffers

// 4-state instance: tiles of NT_NUC4 / pattern_lanes (K) patterns; the five launched 4-state kernels of its K are
// opted in to their dynamic shared memory.  The resident kernel may serve the instance if its whole grid (tiles x
// maxEval) fits the device at once -- every CTA must be running for a job to complete; if it cannot be opted in or
// its occupancy cannot be queried, the instance keeps its launches
int nuc4Setup (Instance *I)
{
    DevCtx &x = I->ctx;
    x.tilePatterns = NT_NUC4 / pattern_lanes (x.K);
    x.patternTiles = x.numTiles = (x.C + x.tilePatterns - 1) / x.tilePatterns;
    return withNuc4K (x.K, [&] (auto k)
        {
        constexpr int KK = decltype (k)::value;
        const int dev = I->cfg.device;
        CK (optIn (eval_nuc4_kernel<KK, NT_NUC4, true>, dev, nuc4Smem<KK, true>));
        CK (optIn (eval_nuc4_kernel<KK, NT_NUC4, false>, dev, nuc4Smem<KK, false>));
        CK (optIn (eval_nuc4_pkernel<KK, NT_NUC4, PARAM_SMALL>, dev, nuc4Smem<KK, true>));
        CK (optIn (eval_nuc4_pkernel<KK, NT_NUC4, PARAM_MID>, dev, nuc4Smem<KK, true>));
        CK (optIn (eval_nuc4_pkernel<KK, NT_NUC4, PARAM_BIG>, dev, nuc4Smem<KK, true>));
        int perSM = 0;
        if (optIn (eval_nuc4_resident_kernel<KK, NT_NUC4>, dev, nuc4Smem<KK, true>) != cudaSuccess ||
            cudaOccupancyMaxActiveBlocksPerMultiprocessor (&perSM, eval_nuc4_resident_kernel<KK, NT_NUC4>, NT_NUC4, nuc4Smem<KK, true>) != cudaSuccess)
            { cudaGetLastError (); perSM = 0; }
        I->res.ok = (long) perSM * I->numSMs >= (long) x.numTiles * I->maxEval;
        return MB200_SUCCESS;
        });
}

// the pipelined tensor-core kernel of S states gets as many operand-ring stages as fit next to its static shared
// memory, and is opted in to the dynamic shared memory they take (stages stays 0 when none fits, or the opt-in is
// refused).  Returns the floats of one pre-split P(t) image.
template <int S>
size_t tcStages (Instance *I)
{
    const int K = I->cfg.category_count;
    int optin = 0;
    cudaDeviceGetAttribute (&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, I->cfg.device);
    cudaFuncAttributes fa;
    const size_t staticBytes = (cudaFuncGetAttributes (&fa, eval_tcp_kernel<S>) == cudaSuccess) ? fa.sharedSizeBytes : 4096;    // barriers, item ring, row maxima
    const size_t limit = ((size_t) optin > staticBytes + 1024) ? (size_t) optin - staticBytes : 0;
    I->tc.stages = tcp_stages<S> (K, limit);
    if (I->tc.stages > 0)
        {
        I->tc.smem = I->tc.stages * tcp_stage_bytes<S> () + tcp_staging_bytes<S> (K) + tcp_tipring_bytes<S> (I->tc.stages);
        if (optIn (eval_tcp_kernel<S>, I->cfg.device, (int) I->tc.smem) != cudaSuccess)
            { cudaGetLastError (); I->tc.stages = 0; }
        }
    return tc_split_floats<S> ();
}

// tensor-core instance: tiles of TC_MIN_ROWS patterns, one persistent CTA per SM; 61 states also opt in
// tiprobs_mm_kernel, which writes the pre-split images
int tensorSetup (Instance *I)
{
    const mb200_instance_config &c = I->cfg;
    DevCtx &x = I->ctx;
    x.tilePatterns = TC_MIN_ROWS;
    x.numTiles = (x.C + TC_MIN_ROWS - 1) / TC_MIN_ROWS;
    int rc = (x.S > 32) ? rcOf (optIn (tiprobs_mm_kernel, c.device, (int) mmSmem (x.S))) : MB200_SUCCESS;
    if (rc) return rc;
    const size_t fl = withTcS (x.S, [&] (auto s) { return tcStages<decltype (s)::value> (I); });
    if (!I->tc.stages) return MB200_ERROR_UNSUPPORTED;          // not for K <= 4 on a 227 KB part
    I->tc.flagStride = (c.partials_count - c.tip_count) + 1;
    rc = zeroed (I->tc.dSplit, (size_t)c.matrix_count * x.K * fl, I->stream);
    if (!rc) rc = zeroed (I->tc.dCounter, 1, I->stream);
    if (!rc) rc = zeroed (I->tc.dError, 1, I->stream);
    if (!rc) rc = zeroed (I->tc.dFlags, (size_t) I->maxEval * (x.numTiles + 1) * I->tc.flagStride, I->stream);
    return rc;
}

// generic instance: TP patterns per tile and KB rate categories per pass of eval_gen_kernel
int genericSetup (Instance *I)
{
    DevCtx &x = I->ctx;
    const int S = x.S, Sp = x.Sp, K = x.K, C = x.C;
    // keep P + child tile + product under ~96 KB
    int TP = 32;
    // rate categories per pass: all of them when their P matrices fit in 48 KB, else one at a time
    const int KB = ((size_t)K * S * (S + 1) * sizeof(float) <= 48*1024) ? K : 1;
    auto smemFor = [&] (int tp) { return sizeof(float) * ((size_t)KB*S*(S+1) + (size_t)KB*tp*(Sp+1) + (size_t)K*tp*S + 3*(size_t)tp); };
    while (TP > 1 && smemFor (TP) > 96*1024) TP >>= 1;
    // small divisions: a CTA walks its tile's nodes one (child, category) step at a time, each step a global round trip and
    // two barriers whatever the tile holds -- fewer patterns per tile put more SMs on the evaluation
    while (TP > 4 && (C + TP - 1) / TP < I->numSMs) TP >>= 1;
    I->smemGen = smemFor (TP);
    x.tilePatterns = TP;
    x.genKB = KB;
    x.numTiles = (C + TP - 1) / TP;
    int rc = (S > 32) ? rcOf (optIn (tiprobs_mm_kernel, I->cfg.device, (int) mmSmem (S))) : MB200_SUCCESS;
    if (!rc && I->smemGen > 48*1024) rc = rcOf (optIn (eval_gen_kernel<NT_GEN>, I->cfg.device, (int) I->smemGen));
    return rc;
}

// variable-state instance: tiles of NT_STD / pattern_lanes (K) patterns
void stdSetup (Instance *I)
{
    DevCtx &x = I->ctx;
    I->vs.sx.lanes = pattern_lanes (x.K);
    x.tilePatterns = NT_STD / I->vs.sx.lanes;
    x.numTiles = (x.C + x.tilePatterns - 1) / x.tilePatterns;
}

// ---- resident generation kernel (eval_nuc4_resident_kernel) ----------------------------------
// A generation of the replay path costs a launch, the time until the kernel starts and the time until
// its results reach the host, all on the critical path, because generation g+1 cannot start before
// the host has read g's lnL.  Instead one kernel stays resident and the host posts each batch to a
// mailbox in mapped host memory.
const unsigned long long RES_IDLE_NS = 100000;   // the kernel exits by itself after this long without a job
const double RES_DEADLINE_S = 10.0;              // longest host wait for the results of a posted job

double wallNow () { struct timespec ts; clock_gettime (CLOCK_MONOTONIC, &ts); return (double) ts.tv_sec + 1e-9 * (double) ts.tv_nsec; }

// write one post: every 16-byte piece carries the sequence number and is written by one aligned
// 16-byte store, so the leader CTA sees each piece whole, from this post or from an earlier one
void post (Instance *I, int seq, int count, const Batch *b)
{
    const int nP = MB200_RES_HEAD + 2 * I->maxEval;
    alignas(16) int4 p[MB200_RES_PIECES];
    memset (p, 0, sizeof(p));
    p[0].x = count;
    if (b)
        {
        const unsigned long long blob = (unsigned long long) b->dBlob.p, res = (unsigned long long) b->hRes.dev;
        p[0].y = (int)(unsigned) blob; p[0].z = (int)(unsigned)(blob >> 32);
        p[1].x = (int)(unsigned) res;  p[1].y = (int)(unsigned)(res >> 32); p[1].z = (int) b->offEval;
        p[2].x = (int) b->offDbl; p[2].y = (int) b->offChunk; p[2].z = (int) b->offCmat;
        p[3].x = (int) b->offOp;
        for (int e = 0; e < b->nEval; e++)
            {
            const JobIndexEntry &je = b->jx.e[e];
            p[MB200_RES_HEAD + 2*e]     = make_int4 (je.matOff, je.nMat, je.opOff, 0);
            p[MB200_RES_HEAD + 2*e + 1] = make_int4 (je.nOp, je.dOff, je.eigen0, 0);
            }
        }
    for (int i = 0; i < nP; i++)
        {
        p[i].w = seq;
        _mm_store_si128 (reinterpret_cast<__m128i *>(I->res.mail.p + i), _mm_load_si128 (reinterpret_cast<const __m128i *>(p + i)));
        }
    __atomic_signal_fence (__ATOMIC_SEQ_CST);
}

// Which batches the resident kernel serves: fused 4-state batches whose evaluations all reach the root,
// whose tile partials the host sums and whose job index covers every evaluation -- and only while this
// instance is the only one on its device, so that idle resident CTAs never hold SMs other analyses
// (many instances, or the partitions of one analysis) launch into.  Kernel timing and throughput mode
// keep their launches.
bool residentEligible (Instance *I, const Batch &b)
{
    const mb200_instance_config &c = I->cfg;
    if (I->family != Family::Nuc4 || !I->res.ok || I->timing || (c.flags & MB200_CONFIG_THROUGHPUT) || !b.fused || !b.allRoot ||
        b.nEval > MB200_JOB_INDEX_MAX || b.jx.n != b.nEval || I->maxEval > MB200_JOB_INDEX_MAX)
        return false;
    if (I->ctx.numTiles > HOSTSUM_MAX_TILES)
        return false;
    {
    std::lock_guard<std::mutex> g (gLock);
    int live = 0;
    for (const Instance *J : gInstances)
        if (J && J->cfg.device == c.device) live++;
    if (live != 1)
        return false;
    }
    if (!I->res.job)
        {
        // mailbox and job copy on first use; without them the instance keeps its launches
        MappedArray<int4> mail; DevArray<ResidentJob> job;
        if (mail.alloc (MB200_RES_PIECES) || job.alloc (1) || rcOf (cudaMemset (job, 0, sizeof(ResidentJob))))
            { I->res.ok = false; return false; }
        memset (mail, 0, sizeof(int4) * MB200_RES_PIECES);
        I->res.mail = std::move (mail); I->res.job = std::move (job);
        }
    return true;
}

// post batch b, launching a resident kernel first when none is running
int residentStart (Instance *I, Batch &b)
{
    if (b.needInv && !I->invMaskValid)
        {
        int rc = retire (I);                           // the mask kernel must not queue behind a resident kernel
        if (rc == MB200_SUCCESS) rc = ensureInvMask (I);
        if (rc != MB200_SUCCESS) return rc;
        }
    // past half the idle timeout the kernel may have exited: a cheap check saves a lost post
    if (I->res.running && wallNow () - I->res.posted > 0.5e-9 * (double) RES_IDLE_NS && cudaStreamQuery (I->stream) == cudaSuccess)
        I->res.running = false;
    DevCtx ctx = I->ctx;
    ctx.hostSum = 1;
    // a new kernel starts past every sequence number an earlier kernel may have left in its job copy
    const int seq0 = I->res.running ? 0 : ++I->seq;
    const int seq = ++I->seq;
    I->res.posted = wallNow ();
    post (I, seq, b.nEval, &b);
    if (!I->res.running)
        {
        const dim3 grid (ctx.numTiles, I->maxEval);
        int rc = withNuc4K (ctx.K, [&] (auto k)
            {
            constexpr int KK = decltype (k)::value;
            eval_nuc4_resident_kernel<KK, NT_NUC4><<<grid, NT_NUC4, nuc4Smem<KK, true>, I->stream>>> (ctx, I->res.mail.dev, I->res.job, seq0, RES_IDLE_NS);
            CK (cudaGetLastError ());
            return MB200_SUCCESS;
            });
        if (rc != MB200_SUCCESS) return rc;
        I->res.running = true;
        I->launchKind[MB200_KERNEL_NUC4]++;
        }
    setPending (I, b, seq, true, true, ctx.numTiles);
    return MB200_SUCCESS;
}

// wait until the kernel has written the pending evaluation's results into the mapped host buffer.  While a
// resident kernel serves the instance the stream never goes idle, so the wait has a wall-clock deadline; an
// idle stream then means the kernel exited on its timeout before its leader took the post, so no CTA
// ran the job and it is posted again to a new kernel.
int waitResults (Instance *I)
{
    const Pending &p = I->pending;             // a relaunch below records the same evaluation with a new seq
    volatile DevResult *r = p.batch->hRes;
    const int slots = p.hostSum ? p.count * p.tiles : p.count;
    unsigned long long spins = 0;
    const double t0 = wallNow ();
    for (int e = 0; e < slots; e++)
        {
        // p.seq: the launch or post begin() issued, whatever else ran on the instance since
        while (r[e].seq != p.seq)
            {
#if defined(__x86_64__)
            __builtin_ia32_pause ();
#endif
            if ((++spins & (I->res.running ? 0x3fffu : 0xfffffu)) == 0)
                {
                cudaError_t q = cudaStreamQuery (I->stream);
                if (q == cudaSuccess)
                    {
                    if (r[e].seq == p.seq) break;
                    if (I->res.running && p.resident)
                        {
                        for (int i = 0; i < slots; i++)
                            if (r[i].seq == p.seq)
                                {
                                fprintf (stderr, "mb200: resident kernel exited in the middle of a job\n");
                                return MB200_ERROR_GENERAL;
                                }
                        I->res.running = false;
                        int rc = residentStart (I, *p.batch);
                        if (rc != MB200_SUCCESS) return rc;
                        e = -1;                 // every slot again, for the new sequence number
                        break;
                        }
                    // stream idle but no result: treat as failure rather than spin forever
                    if (spins > (1ull << 26)) return MB200_ERROR_GENERAL;
                    }
                else if (q != cudaErrorNotReady)
                    {
                    fprintf (stderr, "mb200: CUDA error %s while waiting for results\n", cudaGetErrorName (q));
                    return MB200_ERROR_CUDA;
                    }
                else if (I->res.running && wallNow () - t0 > RES_DEADLINE_S)
                    {
                    fprintf (stderr, "mb200: no results from the resident kernel within %.0f s\n", RES_DEADLINE_S);
                    return MB200_ERROR_GENERAL;
                    }
                }
            }
        }
    // the lnL / status words are ordinary loads: order them after the sequence-number polls
    __atomic_thread_fence (__ATOMIC_ACQUIRE);
    return MB200_SUCCESS;
}

// stop the resident kernel (if any) and wait for it to exit; a job still pending is collected first,
// so that the stop does not overwrite a post the leader has not taken yet
int retire (Instance *I)
{
    if (!I->res.running)
        return MB200_SUCCESS;
    if (I->pending.count > 0 && I->pending.resident)
        {
        int rc = waitResults (I);
        if (rc != MB200_SUCCESS) return rc;
        }
    I->res.running = false;
    post (I, ++I->seq, MB200_RES_STOP, nullptr);
    CK (cudaStreamSynchronize (I->stream));     // bounded: the leader takes the stop within microseconds, or has exited
    return MB200_SUCCESS;
}

// first half of an evaluation: validate, pack, launch.  Returns as soon as the work is queued.
int runBegin (Instance *I, const mb200_evaluation *evs, int count)
{
    if (I->pending.count > 0)
        return MB200_ERROR_OUT_OF_RANGE;               // one evaluation in flight per instance
    Batch &b = I->scratch;
    int rc = pack (I, b, evs, count);
    if (rc != MB200_SUCCESS) return rc;
    const bool viaParams = paramEligible (I, b);
    if (!viaParams)
        CK (cudaMemcpyAsync (b.dBlob, b.hBlob, b.bytes, cudaMemcpyHostToDevice, I->stream));
    return launch (I, b, viaParams, true);
}

// second half: wait for the results of the pending evaluation
int runEnd (Instance *I, double *lnL, int *status)
{
    if (I->pending.count <= 0)
        return MB200_ERROR_OUT_OF_RANGE;
    const Pending p = I->pending;                      // a relaunch inside the wait changes only its seq
    const Batch &b = *p.batch;
    // results land in pinned host memory; no D2H copy, no stream synchronisation
    const int rc = b.allRoot ? waitResults (I) : MB200_SUCCESS;
    I->pending = Pending ();
    if (rc != MB200_SUCCESS) return rc;
    if (!b.allRoot)
        CK (cudaStreamSynchronize (I->stream));
    for (int e = 0; e < p.count; e++)
        {
        if (b.hasRoot[e])
            {
            if (p.hostSum)
                {
                // the tiles' partial sums, added left to right (the order the device uses too)
                double tot = 0.0; int ab = 0;
                for (int t = 0; t < p.tiles; t++)
                    {
                    tot += b.hRes[e * p.tiles + t].lnL;
                    ab  |= b.hRes[e * p.tiles + t].status;
                    }
                if (lnL)    lnL[e] = ab ? -DBL_MAX : tot;
                if (status) status[e] = ab ? MB200_EVAL_UNDERFLOW : MB200_EVAL_OK;
                }
            else
                {
                if (lnL)    lnL[e] = b.hRes[e].lnL;
                if (status) status[e] = b.hRes[e].status;
                }
            }
        else
            {
            if (lnL)    lnL[e] = 0.0;
            if (status) status[e] = MB200_EVAL_OK;
            }
        }
    if (I->eig.status && *(volatile int *) I->eig.status.p != 0)
        {
        // an eigensystem this launch (or an earlier one) read did not converge: nothing computed from it can be used
        *(volatile int *) I->eig.status.p = 0;
        fprintf (stderr, "mb200: device eigensolver did not converge\n");
        return MB200_ERROR_GENERAL;
        }
    return MB200_SUCCESS;
}

int runSync (Instance *I, const mb200_evaluation *evs, int count, double *lnL, int *status)
{
    int rc = runBegin (I, evs, count);
    if (rc != MB200_SUCCESS) return rc;
    return runEnd (I, lnL, status);
}

// the eigensolver's staging into `out`, complete, or an error and `out` unchanged
int makeEigenSolver (const Instance *I, EigenSolver &out)
{
    EigenSolver g;
    const int S = I->cfg.state_count, parts = I->cijkParts, slots = I->cfg.eigen_count;
    const size_t n2 = (size_t)S * S, N = (S + 1) & ~1;
    g.inStride = (size_t)parts * n2 + S;
    int rc = g.dIn.alloc (slots * g.inStride);
    if (!rc) rc = g.hIn.alloc (slots * g.inStride);
    if (!rc) rc = g.status.alloc (1);
    if (!rc && !I->dFactor) rc = g.vec.alloc ((size_t)slots * parts * 2 * n2);
    if (!rc) rc = g.U.alloc ((size_t)slots * parts * N * N);
    if (!rc) rc = g.log.alloc ((size_t)parts * MB200_EIG_LOG_DOUBLES / 2);
    if (!rc) rc = g.rounds.alloc (parts);
    if (!rc) rc = makeEvents (g.evIn, slots, cudaEventDisableTiming);
    if (!rc) rc = rcOf (optIn (eigen_rotations_kernel, I->cfg.device, (int) eigen_smem_bytes ()));
    if (rc != MB200_SUCCESS) return rc;
    *g.status.p = 0;
    g.warmChain.assign (slots, -1);
    out = std::move (g);
    return MB200_SUCCESS;
}

void destroy (Instance *I)
{
    cudaSetDevice (I->cfg.device);
    retire (I);
    if (I->stream) cudaStreamSynchronize (I->stream);
    delete I;
}

} // namespace

extern "C" {

int mb200_abi_version (void) { return MB200_ABI_VERSION; }

const char *mb200_version_string (void) { return "mb200 0.1 (sm_90a)"; }

const char *mb200_error_string (int code)
{
    switch (code)
        {
        case MB200_SUCCESS:             return "success";
        case MB200_ERROR_GENERAL:       return "general error";
        case MB200_ERROR_OUT_OF_MEMORY: return "out of device memory";
        case MB200_ERROR_OUT_OF_RANGE:  return "index or size out of range";
        case MB200_ERROR_NO_DEVICE:     return "no sm_90 (H100) device available; the engine has no CPU fallback";
        case MB200_ERROR_UNSUPPORTED:   return "unsupported configuration";
        case MB200_ERROR_BAD_INSTANCE:  return "bad instance handle";
        case MB200_ERROR_CUDA:          return "CUDA runtime error";
        default:                        return "unknown error";
        }
}

int mb200_device_count (void)
{
    int n = 0, ok = 0;
    if (cudaGetDeviceCount (&n) != cudaSuccess)
        { cudaGetLastError (); return 0; }
    for (int d = 0; d < n; d++)
        {
        int major = 0;
        if (cudaDeviceGetAttribute (&major, cudaDevAttrComputeCapabilityMajor, d) == cudaSuccess && major == 9)
            ok++;
        }
    return ok;
}

int mb200_create_instance (const mb200_instance_config *cfg, int *instance)
{
    if (!cfg || !instance)
        return MB200_ERROR_GENERAL;
    *instance = -1;
    if (cfg->state_count < 2 || cfg->state_count > MB200_MAX_STATES ||
        cfg->category_count < 1 || cfg->category_count > MB200_MAX_CATEGORIES ||
        cfg->pattern_count < 1 || cfg->tip_count < 2 || cfg->partials_count <= cfg->tip_count ||
        cfg->matrix_count < 1 || cfg->scaler_count < 1 || cfg->eigen_count < 1 || cfg->weight_rows < 1)
        return MB200_ERROR_OUT_OF_RANGE;

    int n = 0;
    if (cudaGetDeviceCount (&n) != cudaSuccess || n < 1)
        { cudaGetLastError (); return MB200_ERROR_NO_DEVICE; }
    if (cfg->device < 0 || cfg->device >= n)
        return MB200_ERROR_NO_DEVICE;
    int major = 0, sms = 0;
    if (cudaDeviceGetAttribute (&major, cudaDevAttrComputeCapabilityMajor, cfg->device) != cudaSuccess || major != 9)
        return MB200_ERROR_NO_DEVICE;        // kernels exist for sm_90a only
    CK (cudaSetDevice (cfg->device));
    cudaDeviceGetAttribute (&sms, cudaDevAttrMultiProcessorCount, cfg->device);

    Instance *I = new Instance ();
    I->cfg = *cfg;
    I->family = familyOf (*cfg);
    I->numSMs = sms > 0 ? sms : 132;
    I->maxEval = cfg->max_evaluations > 0 ? cfg->max_evaluations : 1;
    const int S = cfg->state_count, K = cfg->category_count, C = cfg->pattern_count;
    const int Sp = (S + 3) & ~3;
    const size_t nInt = (size_t)(cfg->partials_count - cfg->tip_count);
    I->cijkParts = ((cfg->flags >> 8) & 0xff) > 1 ? ((cfg->flags >> 8) & 0xff) : 1;
    if (I->cijkParts != 1 && (I->cijkParts != K || S == 4)) { delete I; return MB200_ERROR_UNSUPPORTED; }
    I->eigenStride = (size_t) I->cijkParts * (2*(size_t)S + (size_t)S*S*S);
    if (I->family == Family::Std && (S > MB200_STD_MAX_STATES || I->cijkParts != 1)) { delete I; return MB200_ERROR_UNSUPPORTED; }
    if (I->family == Family::Nuc4 && (nInt * K * C >= (1ull << 32) || (size_t)cfg->tip_count * C >= (1ull << 32)))
        { delete I; return MB200_ERROR_OUT_OF_RANGE; }      // 4-state records carry 32-bit element offsets (64 GB of partials)

    DevCtx &x = I->ctx;
    memset (&x, 0, sizeof(x));
    x.S = S; x.Sp = Sp; x.K = K; x.C = C;
    x.tipCount = cfg->tip_count; x.partialsCount = cfg->partials_count; x.matrixCount = cfg->matrix_count;
    x.scalerCount = cfg->scaler_count; x.eigenCount = cfg->eigen_count; x.weightRows = cfg->weight_rows;
    x.cijkParts = I->cijkParts;

    int rc = rcOf (cudaStreamCreateWithFlags (&I->stream.h, cudaStreamNonBlocking));
    if (!rc && S > 32) rc = zeroed (I->dFactor, (size_t)cfg->eigen_count * I->cijkParts * 2 * S * S, I->stream);
    if (!rc)
        switch (I->family)
            {
            case Family::Nuc4:    rc = nuc4Setup (I); break;
            case Family::Tensor:  rc = tensorSetup (I); break;
            case Family::Generic: rc = genericSetup (I); break;
            case Family::Std:     stdSetup (I); break;
            }
    // tile partials per evaluation: the tensor family's buffers, like its flags, hold one tile more than its kernel uses
    const size_t tileSlots = (size_t) I->maxEval * (x.numTiles + (I->family == Family::Tensor ? 1 : 0));
    if (!rc) rc = zeroed (I->dTip8,     (size_t)cfg->tip_count * C, I->stream);
    if (!rc) rc = zeroed (I->dTip64,    (size_t)cfg->tip_count * C, I->stream);
    if (!rc) rc = zeroed (I->dTipPartAmbig, (size_t)cfg->tip_count, I->stream);
    if (!rc) rc = zeroed (I->dPartials, nInt * K * C * Sp, I->stream);
    if (!rc) rc = zeroed (I->dMatrices, (size_t)cfg->matrix_count * K * S * S, I->stream);
    if (!rc) rc = zeroed (I->dScalers,  (size_t)cfg->scaler_count * C, I->stream);
    if (!rc) rc = zeroed (I->dWeights,  (size_t)cfg->weight_rows * C, I->stream);
    if (!rc) rc = zeroed (I->dEigen,    (size_t)cfg->eigen_count * I->eigenStride, I->stream);
    if (!rc) rc = zeroed (I->dInvMask,  (size_t)C, I->stream);
    if (!rc) rc = zeroed (I->dTilePartial, tileSlots, I->stream);
    if (!rc) rc = zeroed (I->dTileAbort,   tileSlots, I->stream);
    if (!rc) rc = zeroed (I->dTicket,      (size_t)I->maxEval, I->stream);
    if (!rc) rc = rcOf (cudaStreamSynchronize (I->stream));
    if (rc != MB200_SUCCESS)
        { destroy (I); return rc; }           // the half-built instance frees what it holds
    I->tipPartAmbig.assign (cfg->tip_count, 0);
    x.tip8 = I->dTip8; x.tip64 = I->dTip64; x.tipPartAmbig = I->dTipPartAmbig; x.partials = I->dPartials; x.matrices = I->dMatrices;
    x.scalers = I->dScalers; x.eigen = I->dEigen; x.weights = I->dWeights; x.invMask = I->dInvMask;
    x.tilePartial = I->dTilePartial; x.tileAbort = I->dTileAbort; x.ticket = I->dTicket;

    std::lock_guard<std::mutex> g (gLock);
    for (size_t i = 0; i < gInstances.size (); i++)
        if (gInstances[i] == nullptr) { gInstances[i] = I; *instance = (int) i; return MB200_SUCCESS; }
    gInstances.push_back (I);
    *instance = (int) gInstances.size () - 1;
    return MB200_SUCCESS;
}

int mb200_finalize_instance (int instance)
{
    Instance *I;
    {
    std::lock_guard<std::mutex> g (gLock);
    if (instance < 0 || instance >= (int) gInstances.size () || !gInstances[instance])
        return MB200_ERROR_BAD_INSTANCE;
    I = gInstances[instance];
    gInstances[instance] = nullptr;
    }
    destroy (I);
    return MB200_SUCCESS;
}

int mb200_set_tip_states (int instance, int tip, const uint64_t *masks)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (tip < 0 || tip >= I->cfg.tip_count || !masks) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const int C = I->cfg.pattern_count;
    std::vector<uint64_t> h64 (C); std::vector<uint8_t> h8 (C);     // pageable: the copies are waited for below
    const uint64_t full = (I->cfg.state_count == 64) ? ~(uint64_t)0 : (((uint64_t)1 << I->cfg.state_count) - 1);
    int partAmbig = 0;      // isPartAmbig of SetUpTermState (src/mcmc.c:18631-18651)
    for (int c = 0; c < C; c++)
        {
        h64[c] = masks[c] & full;
        h8[c]  = (uint8_t)(h64[c] & 0xff);
        if (h64[c] != full && (h64[c] == 0 || (h64[c] & (h64[c] - 1)) != 0))
            partAmbig = 1;
        }
    CK (cudaMemcpyAsync (I->dTipPartAmbig + tip, &partAmbig, sizeof(int), cudaMemcpyHostToDevice, I->stream));
    I->tipPartAmbig[tip] = partAmbig;
    I->tipEpoch++;                  // packed 4-state batches carry the tip kinds: re-pack after this
    CK (cudaMemcpyAsync (I->dTip64 + (size_t)tip * C, h64.data (), (size_t)C * 8, cudaMemcpyHostToDevice, I->stream));
    CK (cudaMemcpyAsync (I->dTip8 + (size_t)tip * C, h8.data (), (size_t)C, cudaMemcpyHostToDevice, I->stream));
    CK (cudaStreamSynchronize (I->stream));
    I->invMaskValid = false;
    return MB200_SUCCESS;
}

int mb200_set_pattern_weights (int instance, int row, const float *w)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (row < 0 || row >= I->cfg.weight_rows || !w) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const int C = I->cfg.pattern_count;
    CK (cudaMemcpyAsync (I->dWeights + (size_t)row * C, w, (size_t)C * sizeof(float), cudaMemcpyHostToDevice, I->stream));
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

int mb200_set_pattern_states (int instance, const int *ns, const int *ti, const int *bs, int matLen, int dummy, int uncompressed)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (I->family != Family::Std) return MB200_ERROR_UNSUPPORTED;
    const int C = I->cfg.pattern_count, K = I->cfg.category_count;
    if (!ns || !ti || !bs || matLen < 1 || dummy < 0 || dummy > C) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    // state-count classes: (n, offset) pairs, every pattern of a class sharing the offset
    std::vector<int2> classes;
    for (int c = 0; c < C; c++)
        {
        if (ns[c] < 2 || ns[c] > I->cfg.state_count || ti[c] < 0 || (long) ti[c] + (long) K * ns[c] * ns[c] > (long) matLen ||
            bs[c] < 0 || bs[c] + ns[c] > MB200_MAX_STATES)
            return MB200_ERROR_OUT_OF_RANGE;
        bool seen = false;
        for (const int2 &q : classes)
            if (q.x == ns[c] && q.y == ti[c]) { seen = true; break; }
        if (!seen)
            {
            if ((int) classes.size () >= MB200_STD_MAX_STATES) return MB200_ERROR_UNSUPPORTED;
            classes.push_back (make_int2 (ns[c], ti[c]));
            }
        }
    // the new tables and matrices (a branch's: one block of matLen floats, m->tiProbLength) are complete before the
    // old ones go: on failure the instance keeps those
    const size_t matFloats = (size_t)I->cfg.matrix_count * matLen;
    DevArray<int> dTab; DevArray<int2> dClasses; DevArray<float> dMats;
    if ((rc = dTab.alloc (3 * (size_t)C)) || (rc = dClasses.alloc (MB200_STD_MAX_STATES)) || (rc = dMats.alloc (matFloats))) return rc;
    CK (cudaMemsetAsync (dMats, 0, matFloats * sizeof(float), I->stream));
    CK (cudaMemcpyAsync (dTab, ns, (size_t)C * sizeof(int), cudaMemcpyHostToDevice, I->stream));
    CK (cudaMemcpyAsync (dTab + C, ti, (size_t)C * sizeof(int), cudaMemcpyHostToDevice, I->stream));
    CK (cudaMemcpyAsync (dTab + 2*(size_t)C, bs, (size_t)C * sizeof(int), cudaMemcpyHostToDevice, I->stream));
    CK (cudaMemcpyAsync (dClasses, classes.data (), classes.size () * sizeof(int2), cudaMemcpyHostToDevice, I->stream));
    CK (cudaStreamSynchronize (I->stream));
    StdTables &v = I->vs;
    v.dTab = std::move (dTab); v.dClasses = std::move (dClasses); I->dMatrices = std::move (dMats);
    I->ctx.matrices = I->dMatrices;
    I->ring = MatRing ();                       // its slots hold matrices of the old length
    v.hNStates.assign (ns, ns + C); v.hTiIndex.assign (ti, ti + C); v.hBsIndex.assign (bs, bs + C);
    v.hClOff.assign (C + 1, 0);
    v.freqLen = 0;
    for (int c = 0; c < C; c++)
        {
        v.hClOff[c + 1] = v.hClOff[c] + (size_t) ns[c];
        if (bs[c] + ns[c] > v.freqLen) v.freqLen = bs[c] + ns[c];
        }
    v.sx.nStates = v.dTab; v.sx.tiIndex = v.dTab + C; v.sx.bsIndex = v.dTab + 2*(size_t)C;
    v.sx.classes = v.dClasses; v.sx.nClasses = (int) classes.size ();
    v.sx.matLen = matLen; v.sx.dummy = dummy; v.sx.uncompressed = uncompressed;
    v.uniformMk = true;
    v.ready = true;
    return MB200_SUCCESS;
}

int mb200_set_cijk (int instance, int eigen, const double *block)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (eigen < 0 || eigen >= I->cfg.eigen_count || !block) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    if (!I->eig.warmChain.empty ()) I->eig.warmChain[eigen] = -1;      // this slot's eigenvectors no longer come from the device solver
    CK (cudaMemcpyAsync (I->dEigen + (size_t)eigen * I->eigenStride, block, I->eigenStride * sizeof(double),
                         cudaMemcpyHostToDevice, I->stream));
    if (I->dFactor)
        {
        const int S = I->cfg.state_count;
        cijk_factor_kernel<<<dim3 (S, I->cijkParts), 256, 0, I->stream>>> (I->dEigen + (size_t)eigen * I->eigenStride,
                                                                            I->dFactor + (size_t)eigen * I->cijkParts * 2 * S * S, S);
        CK (cudaGetLastError ());
        I->launchKind[MB200_KERNEL_SETUP]++;
        }
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

int mb200_set_eigen_decomposition (int instance, int eigen, const double *V, const double *Vinv, const double *lambda)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (eigen < 0 || eigen >= I->cfg.eigen_count || !V || !Vinv || !lambda) return MB200_ERROR_OUT_OF_RANGE;
    if (I->cijkParts != 1) return MB200_ERROR_UNSUPPORTED;        // multi-part slots are uploaded whole (mb200_set_cijk)
    int rc = use (I); if (rc) return rc;
    if (!I->eig.warmChain.empty ()) I->eig.warmChain[eigen] = -1;
    const int S = I->cfg.state_count;
    const size_t n2 = (size_t)S * S;
    DevArray<double> tmp;                   // freed on return, after the stream has been waited for
    if ((rc = tmp.alloc (2*n2 + S))) return rc;
    CK (cudaMemcpyAsync (tmp, V, n2 * sizeof(double), cudaMemcpyHostToDevice, I->stream));
    CK (cudaMemcpyAsync (tmp + n2, Vinv, n2 * sizeof(double), cudaMemcpyHostToDevice, I->stream));
    CK (cudaMemcpyAsync (tmp + 2*n2, lambda, (size_t)S * sizeof(double), cudaMemcpyHostToDevice, I->stream));
    size_t n3 = n2 * S;
    int blocks = (int)((n3 + 255) / 256); if (blocks > 1024) blocks = 1024;
    cijk_kernel<<<blocks, 256, 0, I->stream>>> (I->dEigen + (size_t)eigen * I->eigenStride, tmp, tmp + n2, tmp + 2*n2, S);
    I->launchKind[MB200_KERNEL_SETUP]++;
    if (I->dFactor)         // the factors are the caller's V and V^-1 themselves
        {
        CK (cudaMemcpyAsync (I->dFactor + (size_t)eigen * 2 * n2, tmp, n2 * sizeof(double), cudaMemcpyDeviceToDevice, I->stream));
        CK (cudaMemcpyAsync (I->dFactor + (size_t)eigen * 2 * n2 + n2, tmp + n2, n2 * sizeof(double), cudaMemcpyDeviceToDevice, I->stream));
        }
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

// Rate matrices in, eigensystems out, all on the instance's stream: nothing here waits for the device.
int mb200_set_rate_matrices (int instance, int eigen, int like_eigen, const double *Q, const double *pi)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (eigen < 0 || eigen >= I->cfg.eigen_count || like_eigen >= I->cfg.eigen_count || !Q || !pi) return MB200_ERROR_OUT_OF_RANGE;
    const int S = I->cfg.state_count, parts = I->cijkParts;
    if (I->family == Family::Std || S < 2 || S > MB200_EIG_NMAX) return MB200_ERROR_UNSUPPORTED;
    for (int s = 0; s < S; s++)
        if (!(pi[s] > 0.0)) return MB200_ERROR_OUT_OF_RANGE;           // sqrt(pi) scales the similarity transform
    int rc = use (I); if (rc) return rc;
    const size_t n2 = (size_t)S * S;
    const int    N = (S + 1) & ~1;
    const size_t uLen = (size_t)parts * N * N;
    if (!I->eig.dIn && (rc = makeEigenSolver (I, I->eig))) return rc;
    EigenSolver &g = I->eig;
    CK (cudaEventSynchronize (g.evIn[eigen]));              // the slot's previous matrices have left the staging area
    double *h = g.hIn + (size_t)eigen * g.inStride, *d = g.dIn + (size_t)eigen * g.inStride;
    memcpy (h, Q, (size_t)parts * n2 * sizeof(double));
    memcpy (h + (size_t)parts * n2, pi, (size_t)S * sizeof(double));
    CK (cudaMemcpyAsync (d, h, g.inStride * sizeof(double), cudaMemcpyHostToDevice, I->stream));
    CK (cudaEventRecord (g.evIn[eigen], I->stream));
    // warm start from the eigenvectors of a nearby matrix, unless that would extend an already long chain of warm starts
    const double *U0 = nullptr;
    int chain = 0;
    if (like_eigen >= 0 && like_eigen != eigen && g.warmChain[like_eigen] >= 0 && g.warmChain[like_eigen] < MB200_EIG_WARM_CHAIN)
        {
        U0 = g.U + (size_t)like_eigen * uLen;
        chain = g.warmChain[like_eigen] + 1;
        }
    g.warmChain[eigen] = chain;
    const double *dPi = d + (size_t)parts * n2;
    double *vec = (I->dFactor ? I->dFactor : g.vec) + (size_t)eigen * parts * 2 * n2, *block = I->dEigen + (size_t)eigen * I->eigenStride;
    eigen_rotations_kernel<<<parts, MB200_EIG_THREADS, eigen_smem_bytes (), I->stream>>> (d, dPi, S, U0, g.log, g.rounds, block, g.status.dev);
    eigen_vectors_kernel<<<dim3 ((N + 7) / 8, parts), 256, 0, I->stream>>> (dPi, S, U0, g.log, g.rounds, g.U + (size_t)eigen * uLen, vec);
    const size_t n3 = n2 * S;
    int blocks = (int)((n3 + 255) / 256); if (blocks > 512) blocks = 512;
    cijk_parts_kernel<<<dim3 (blocks, parts), 256, 0, I->stream>>> (block, vec, S);
    CK (cudaGetLastError ());
    I->launchKind[MB200_KERNEL_SETUP] += 3;
    return MB200_SUCCESS;
}

int mb200_update_transition_matrices (int instance, const mb200_matrix_update *updates, int count,
                                      const double *category_rates, const double *state_freqs)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    // stationary rows (t > TIME_MAX) are the frequencies: only the variable-state family, whose Mk matrices do not
    // read them, may leave them out
    if (count < 0 || (count > 0 && !updates) || !category_rates || (!state_freqs && I->family != Family::Std))
        return MB200_ERROR_OUT_OF_RANGE;
    if (count == 0) return MB200_SUCCESS;
    int rc = use (I); if (rc) return rc;
    mb200_evaluation ev;
    memset (&ev, 0, sizeof(ev));
    ev.matrix_update_count = count; ev.matrix_updates = updates;
    ev.site_scaler_dst = MB200_NONE; ev.site_scaler_src = MB200_NONE; ev.root_buffer = MB200_NONE;
    for (int k = 0; k < I->cfg.category_count; k++) { ev.category_rates[k] = category_rates[k]; ev.category_weights[k] = 1.0; }
    if (state_freqs)
        for (int s = 0; s < I->cfg.state_count; s++) ev.state_freqs[s] = state_freqs[s];
    return runSync (I, &ev, 1, nullptr, nullptr);
}

int mb200_update_partials (int instance, const mb200_operation *operations, int count, int site_scaler)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (count < 0 || (count > 0 && !operations)) return MB200_ERROR_OUT_OF_RANGE;
    if (count == 0) return MB200_SUCCESS;
    int rc = use (I); if (rc) return rc;
    mb200_evaluation ev;
    memset (&ev, 0, sizeof(ev));
    ev.operation_count = count; ev.operations = operations;
    ev.site_scaler_dst = site_scaler; ev.site_scaler_src = site_scaler; ev.root_buffer = MB200_NONE;
    for (int k = 0; k < I->cfg.category_count; k++) ev.category_weights[k] = 1.0;
    return runSync (I, &ev, 1, nullptr, nullptr);
}

int mb200_reset_scalers (int instance, int scaler)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (scaler < 0 || scaler >= I->cfg.scaler_count) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const int C = I->cfg.pattern_count;
    CK (cudaMemsetAsync (I->dScalers + (size_t)scaler * C, 0, (size_t)C * sizeof(float), I->stream));
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

int mb200_copy_scalers (int instance, int dst, int src)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (dst < 0 || dst >= I->cfg.scaler_count || src < 0 || src >= I->cfg.scaler_count) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const int C = I->cfg.pattern_count;
    CK (cudaMemcpyAsync (I->dScalers + (size_t)dst * C, I->dScalers + (size_t)src * C, (size_t)C * sizeof(float),
                         cudaMemcpyDeviceToDevice, I->stream));
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

int mb200_root_log_likelihood (int instance, int root_buffer, int site_scaler, int weights_row,
                               const double *state_freqs, const double *category_weights, int has_p_invar,
                               double p_invar, int flags, double *lnL, int *status)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (!state_freqs || !category_weights || !lnL) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    mb200_evaluation ev;
    memset (&ev, 0, sizeof(ev));
    ev.site_scaler_dst = MB200_NONE; ev.site_scaler_src = site_scaler; ev.root_buffer = root_buffer;
    ev.weights_row = weights_row; ev.flags = flags; ev.has_p_invar = has_p_invar; ev.p_invar = p_invar;
    for (int k = 0; k < I->cfg.category_count; k++) ev.category_weights[k] = category_weights[k];
    // variable-state divisions: the whole table the patterns index (freq_offsets[c] + state_counts[c]), which may
    // be longer than state_count
    const int nFreq = (I->family == Family::Std) ? I->vs.freqLen : I->cfg.state_count;
    for (int s = 0; s < nFreq; s++) ev.state_freqs[s] = state_freqs[s];
    int st = 0;
    rc = runSync (I, &ev, 1, lnL, &st);
    if (status) *status = st;
    return rc;
}

int mb200_evaluate (int instance, const mb200_evaluation *evaluations, int count, double *lnL, int *status)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (!evaluations || !lnL || !status) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    return runSync (I, evaluations, count, lnL, status);
}

int mb200_evaluate_begin (int instance, const mb200_evaluation *evaluations, int count)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (!evaluations) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    return runBegin (I, evaluations, count);
}

int mb200_evaluate_end (int instance, double *lnL, int *status)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (!lnL || !status) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    return runEnd (I, lnL, status);
}

// ---- read-back / seeding ---------------------------------------------------------------
int mb200_get_partials (int instance, int buffer, float *out)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (!okPartials (I, buffer, false) || !out) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const int S = I->cfg.state_count, K = I->cfg.category_count, C = I->cfg.pattern_count, Sp = I->ctx.Sp;
    const size_t n = (size_t)K * C * Sp;
    std::vector<float> tmp (n);
    CK (cudaMemcpyAsync (tmp.data (), I->dPartials + (size_t)(buffer - I->cfg.tip_count) * n, n * sizeof(float),
                         cudaMemcpyDeviceToHost, I->stream));
    CK (cudaStreamSynchronize (I->stream));
    if (I->family == Family::Std)
        {
        const StdTables &v = I->vs;
        if (!v.ready) return MB200_ERROR_UNSUPPORTED;
        const size_t numReps = v.hClOff[C];                 // ragged [k][c][nStates[c]] (src/likelihood.c:1941-1943)
        for (int k = 0; k < K; k++)
            for (int c = 0; c < C; c++)
                for (int s = 0; s < v.hNStates[c]; s++)
                    out[(size_t)k * numReps + v.hClOff[c] + s] = tmp[((size_t)k * C + c) * Sp + s];
        return MB200_SUCCESS;
        }
    for (size_t r = 0; r < (size_t)K * C; r++)
        for (int s = 0; s < S; s++)
            out[r * S + s] = tmp[r * Sp + s];
    return MB200_SUCCESS;
}

int mb200_set_partials (int instance, int buffer, const float *in)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (!okPartials (I, buffer, false) || !in) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const int S = I->cfg.state_count, K = I->cfg.category_count, C = I->cfg.pattern_count, Sp = I->ctx.Sp;
    const size_t n = (size_t)K * C * Sp;
    std::vector<float> tmp (n, 0.0f);
    if (I->family == Family::Std)
        {
        const StdTables &v = I->vs;
        if (!v.ready) return MB200_ERROR_UNSUPPORTED;
        const size_t numReps = v.hClOff[C];
        for (int k = 0; k < K; k++)
            for (int c = 0; c < C; c++)
                for (int s = 0; s < v.hNStates[c]; s++)
                    tmp[((size_t)k * C + c) * Sp + s] = in[(size_t)k * numReps + v.hClOff[c] + s];
        }
    else
    for (size_t r = 0; r < (size_t)K * C; r++)
        for (int s = 0; s < S; s++)
            tmp[r * Sp + s] = in[r * S + s];
    CK (cudaMemcpyAsync (I->dPartials + (size_t)(buffer - I->cfg.tip_count) * n, tmp.data (), n * sizeof(float),
                         cudaMemcpyHostToDevice, I->stream));
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

int mb200_get_transition_matrix (int instance, int matrix, float *out)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (matrix < 0 || matrix >= I->cfg.matrix_count || !out) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const bool isStd = (I->family == Family::Std);
    if (isStd && !I->vs.ready) return MB200_ERROR_UNSUPPORTED;
    const size_t n = isStd ? (size_t) I->vs.sx.matLen : (size_t)I->cfg.category_count * I->cfg.state_count * I->cfg.state_count;
    CK (cudaMemcpyAsync (out, I->dMatrices + (size_t)matrix * n, n * sizeof(float), cudaMemcpyDeviceToHost, I->stream));
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

int mb200_set_transition_matrix (int instance, int matrix, const float *in)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (matrix < 0 || matrix >= I->cfg.matrix_count || !in) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const bool isStd = (I->family == Family::Std);
    if (isStd && !I->vs.ready) return MB200_ERROR_UNSUPPORTED;
    const size_t n = isStd ? (size_t) I->vs.sx.matLen : (size_t)I->cfg.category_count * I->cfg.state_count * I->cfg.state_count;
    if (isStd) I->vs.uniformMk = false;        // a caller-supplied matrix need not have the Mk form: read every entry from now on
    const bool tensor = (I->family == Family::Tensor);
    const int MAT_RING = 64;
    if (!tensor && n * sizeof(float) <= 64*1024)
        {
        // small matrices (host-built P(t) of a STANDARD division, one call per dirty branch): stage through a pinned ring and let
        // the copy ride the instance's stream -- the evaluation that reads the matrix is queued behind it; no host wait
        if (I->ring.stride < n)                                 // none yet (mb200_set_pattern_states drops it)
            {
            MatRing r;
            if ((rc = r.buf.alloc ((size_t)MAT_RING * n)) || (rc = makeEvents (r.ev, MAT_RING, cudaEventDisableTiming))) return rc;
            r.stride = n;
            I->ring = std::move (r);
            }
        const int slot = I->ring.next++ % MAT_RING;
        CK (cudaEventSynchronize (I->ring.ev[slot]));           // the slot's previous copy has left the ring
        float *h = I->ring.buf + (size_t)slot * I->ring.stride;
        memcpy (h, in, n * sizeof(float));
        CK (cudaMemcpyAsync (I->dMatrices + (size_t)matrix * n, h, n * sizeof(float), cudaMemcpyHostToDevice, I->stream));
        CK (cudaEventRecord (I->ring.ev[slot], I->stream));
        return MB200_SUCCESS;
        }
    CK (cudaMemcpyAsync (I->dMatrices + (size_t)matrix * n, in, n * sizeof(float), cudaMemcpyHostToDevice, I->stream));
    if (tensor)
        {
        const int K = I->cfg.category_count;
        withTcS (I->cfg.state_count, [&] (auto s)
            {
            tc_split_kernel<decltype (s)::value><<<dim3 (1, K), 128, 0, I->stream>>> (I->dMatrices, I->tc.dSplit, nullptr, matrix, K);
            });
        I->launchKind[MB200_KERNEL_SETUP]++;
        }
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

int mb200_get_scalers (int instance, int scaler, float *out)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (scaler < 0 || scaler >= I->cfg.scaler_count || !out) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const int C = I->cfg.pattern_count;
    CK (cudaMemcpyAsync (out, I->dScalers + (size_t)scaler * C, (size_t)C * sizeof(float), cudaMemcpyDeviceToHost, I->stream));
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

int mb200_set_scalers (int instance, int scaler, const float *in)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (scaler < 0 || scaler >= I->cfg.scaler_count || !in) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    const int C = I->cfg.pattern_count;
    CK (cudaMemcpyAsync (I->dScalers + (size_t)scaler * C, in, (size_t)C * sizeof(float), cudaMemcpyHostToDevice, I->stream));
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

// ---- device-resident replay ---------------------------------------------------------------
int mb200_pack_evaluations (int instance, const mb200_evaluation *evaluations, int count, int *batch)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (!evaluations || !batch) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    auto b = std::make_unique<Batch> ();
    rc = pack (I, *b, evaluations, count);
    if (rc != MB200_SUCCESS) return rc;
    if (cudaMemcpyAsync (b->dBlob, b->hBlob, b->bytes, cudaMemcpyHostToDevice, I->stream) != cudaSuccess ||
        cudaStreamSynchronize (I->stream) != cudaSuccess)
        return MB200_ERROR_CUDA;
    size_t i = 0;
    while (i < I->batches.size () && I->batches[i]) i++;
    if (i == I->batches.size ()) I->batches.emplace_back ();
    I->batches[i] = std::move (b);
    *batch = (int) i;
    return MB200_SUCCESS;
}

int mb200_replay (int instance, int batch)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (batch < 0 || batch >= (int) I->batches.size () || !I->batches[batch]) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    Batch &rb = *I->batches[batch];
    if (rb.tipEpoch != I->tipEpoch)
        return MB200_ERROR_OUT_OF_RANGE;           // tip states changed since mb200_pack_evaluations: pack again
    return launch (I, rb, false, false);
}

int mb200_replay_begin (int instance, int batch)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (batch < 0 || batch >= (int) I->batches.size () || !I->batches[batch]) return MB200_ERROR_OUT_OF_RANGE;
    if (I->pending.count > 0) return MB200_ERROR_OUT_OF_RANGE;      // one evaluation in flight per instance
    CK (cudaSetDevice (I->cfg.device));                               // not use (): a resident kernel stays
    Batch &rb = *I->batches[batch];
    if (rb.tipEpoch != I->tipEpoch)
        return MB200_ERROR_OUT_OF_RANGE;
    if (residentEligible (I, rb))
        return residentStart (I, rb);
    int rc = retire (I);
    if (rc != MB200_SUCCESS) return rc;
    return launch (I, rb, false, true);
}

int mb200_replay_end (int instance, double *lnL, int *status)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (!lnL || !status) return MB200_ERROR_OUT_OF_RANGE;
    CK (cudaSetDevice (I->cfg.device));
    return runEnd (I, lnL, status);
}

int mb200_replay_results (int instance, int batch, double *lnL, int *status)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (batch < 0 || batch >= (int) I->batches.size () || !I->batches[batch]) return MB200_ERROR_OUT_OF_RANGE;
    int rc = use (I); if (rc) return rc;
    Batch &b = *I->batches[batch];
    CK (cudaStreamSynchronize (I->stream));
    CK (cudaMemcpy (b.hRes, b.dRes, sizeof(DevResult) * b.nEval, cudaMemcpyDeviceToHost));
    for (int e = 0; e < b.nEval; e++)
        {
        if (lnL) lnL[e] = b.hRes[e].lnL;
        if (status) status[e] = b.hRes[e].status;
        }
    return MB200_SUCCESS;
}

int mb200_free_batch (int instance, int batch)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    if (batch < 0 || batch >= (int) I->batches.size () || !I->batches[batch]) return MB200_ERROR_OUT_OF_RANGE;
    if (I->pending.count > 0 && I->pending.batch == I->batches[batch].get ())
        return MB200_ERROR_OUT_OF_RANGE;          // the pending evaluation writes its results there
    int rc = use (I); if (rc) return rc;
    CK (cudaStreamSynchronize (I->stream));
    I->batches[batch].reset ();
    return MB200_SUCCESS;
}

int mb200_synchronize (int instance)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    int rc = use (I); if (rc) return rc;
    CK (cudaStreamSynchronize (I->stream));
    return MB200_SUCCESS;
}

int mb200_get_stream (int instance, void **stream)
{
    Instance *I = get (instance);
    if (!I || !stream) return MB200_ERROR_BAD_INSTANCE;
    *stream = (void *) I->stream;
    return MB200_SUCCESS;
}

int mb200_get_launch_count (int instance, long long *launches)
{
    Instance *I = get (instance);
    if (!I || !launches) return MB200_ERROR_BAD_INSTANCE;
    *launches = 0;
    for (long long n : I->launchKind) *launches += n;
    return MB200_SUCCESS;
}

int mb200_get_kernel_launches (int instance, int kind, long long *launches)
{
    Instance *I = get (instance);
    if (!I || !launches) return MB200_ERROR_BAD_INSTANCE;
    if (kind < 0 || kind >= MB200_KERNEL_COUNTERS) return MB200_ERROR_OUT_OF_RANGE;
    *launches = (kind < MB200_KERNEL_KINDS) ? I->launchKind[kind] : I->launchNuc4Sub[kind - MB200_KERNEL_KINDS];
    return MB200_SUCCESS;
}

int mb200_set_kernel_timing (int instance, int enabled)
{
    Instance *I = get (instance);
    if (!I) return MB200_ERROR_BAD_INSTANCE;
    int rc = use (I); if (rc) return rc;
    CK (cudaStreamSynchronize (I->stream));
    if (enabled && I->evA.empty ())
        {
        std::vector<Event> a, b;
        if ((rc = makeEvents (a, EV_RING, cudaEventDefault)) || (rc = makeEvents (b, EV_RING, cudaEventDefault))) return rc;
        I->evA = std::move (a); I->evB = std::move (b);
        }
    I->timing = enabled != 0;
    I->evCount = 0;
    return MB200_SUCCESS;
}

int mb200_get_kernel_time (int instance, double *milliseconds, int *launches)
{
    Instance *I = get (instance);
    if (!I || !milliseconds || !launches) return MB200_ERROR_BAD_INSTANCE;
    int rc = use (I); if (rc) return rc;
    CK (cudaStreamSynchronize (I->stream));
    long long n = I->evCount < EV_RING ? I->evCount : EV_RING;
    double tot = 0.0;
    for (long long i = 0; i < n; i++)
        {
        float ms = 0.0f;
        CK (cudaEventElapsedTime (&ms, I->evA[i], I->evB[i]));
        tot += ms;
        }
    *milliseconds = tot;
    *launches = (int) n;
    I->evCount = 0;
    return MB200_SUCCESS;
}

} // extern "C"
