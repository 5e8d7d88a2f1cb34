/*
 * mb200.h -- C-ABI of the H100-native tree-likelihood engine for MrBayes.
 *
 * Plain C, plain pointers and sizes, no torch / CUDA types.  The library
 * (libmb200.so) owns every floating-point buffer of a data division on one
 * GPU; the caller owns all integer bookkeeping and addresses the buffers by
 * the same integer indices MrBayes keeps in ModelInfo (condLikeIndex,
 * tiProbsIndex, nodeScalerIndex, siteScalerIndex, cijkIndex and their
 * *ScratchIndex twins, reference src/bayes.h:1374-1385).  Accept / reject is
 * therefore a pure host-side index swap (ResetFlips, src/mcmc.c:15695-15765)
 * that the engine never sees.
 *
 * What each entry point replaces in the reference (file:line under
 * /root/reference):
 *
 *   mb200_create_instance        createBeagleInstance / InitBeagleInstance
 *                                (src/mbbeagle.c:60-395) and the buffer
 *                                allocation of InitChainCondLikes
 *                                (src/mcmc.c:5703-6508)
 *   mb200_set_tip_states         tip partial fill from parsSets
 *                                (src/mcmc.c:6302-6413), beagleSetTipStates /
 *                                beagleSetTipPartials (src/mbbeagle.c:123-166)
 *   mb200_set_pattern_weights    numSitesOfPat rows (src/mcmc.c:4188,
 *                                src/likelihood.c:5830)
 *   mb200_set_cijk               the cijk block written by UpDateCijk /
 *                                CalcCijk (src/likelihood.c:10476,
 *                                src/utils.c:9734)
 *   mb200_set_eigen_decomposition  beagleSetEigenDecomposition
 *                                (src/likelihood.c:10652)
 *   mb200_set_rate_matrices      GetEigens + CalcCijk inside UpDateCijk
 *                                (src/likelihood.c:10626-10760, src/utils.c:11201)
 *   mb200_update_transition_matrices  TiProbs_Gen (src/likelihood.c:9424) /
 *                                TreeTiProbs_Beagle (src/mbbeagle.c:1368)
 *   mb200_update_partials        CondLikeDown_* / CondLikeRoot_* /
 *                                CondLikeScaler_* / RemoveNodeScalers
 *                                (src/likelihood.c:204-5610, 7981) and
 *                                TreeCondLikes_Beagle_Always_Rescale
 *                                (src/mbbeagle.c:995)
 *   mb200_root_log_likelihood    Likelihood_NUC4* / Likelihood_Gen*
 *                                (src/likelihood.c:5764-6960) /
 *                                TreeLikelihood_Beagle (src/mbbeagle.c:1117)
 *   mb200_set_pattern_states     m->nStates / tiIndex / bsIndex of STANDARD-data
 *                                divisions (src/bayes.h:1329-1331); the *_Std
 *                                kernel family (src/likelihood.c:1920, 4496,
 *                                5547, 7359, 10066)
 *   mb200_evaluate               one whole LaunchLogLikeForDivision
 *                                (src/likelihood.c:7851-7973) per element,
 *                                any number of chains per call, ONE fused
 *                                launch (the chain-batched generation of
 *                                SURVEY.md section 8f-1)
 *
 * Every function returns MB200_SUCCESS (0) or a negative MB200_ERROR_* code;
 * there is no CPU fallback: without a usable sm_90 device
 * mb200_create_instance fails with MB200_ERROR_NO_DEVICE.
 */
#ifndef MB200_H_
#define MB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MB200_ABI_VERSION 1

/* return codes */
#define MB200_SUCCESS                 0
#define MB200_ERROR_GENERAL          -1
#define MB200_ERROR_OUT_OF_MEMORY    -2
#define MB200_ERROR_OUT_OF_RANGE     -3
#define MB200_ERROR_NO_DEVICE        -4
#define MB200_ERROR_UNSUPPORTED      -5
#define MB200_ERROR_BAD_INSTANCE     -6
#define MB200_ERROR_CUDA             -7

/* per-evaluation status written by mb200_evaluate / mb200_root_log_likelihood */
#define MB200_EVAL_OK                 0
/* some pattern had like < LIKE_EPSILON (1e-300): lnL = -DBL_MAX and the caller
 * must set abortMove = YES (src/likelihood.c:44, 5852-5860) */
#define MB200_EVAL_UNDERFLOW          1

#define MB200_MAX_STATES             64   /* numModelStates; 61-state codon fits   */
#define MB200_MAX_CATEGORIES         20   /* MAX_RATE_CATS (src/bayes.h:316)       */
#define MB200_NONE                  (-1)  /* "no buffer" sentinel, like BEAGLE_OP_NONE */
#define MB200_EIGEN_INLINE          (-2)  /* mb200_matrix_update.eigen: use mb200_evaluation.inline_eigen */

/* instance flags.  Models whose categories have their own rate matrices (codon NY98 / M3: one
 * eigensystem per omega category, m->nCijkParts = numOmegaCats, TiProbs_GenCov,
 * src/likelihood.c:9568) keep `parts` consecutive [2S + S^3] blocks per cijk slot, the layout of
 * m->cijks[] (cijkLength = parts * (2S + S^3)); category k uses part k.  parts must be 1 or equal to
 * category_count. */
#define MB200_CONFIG_CIJK_PARTS(n) (((n) & 0xff) << 8)
/* Favour throughput over the latency of one call: set it when several instances (independent
 * analyses, or the partitions of a large data set) keep the GPU busy together.  4-state path: one
 * CTA per evaluation walks all pattern tiles and rebuilds P(t) once instead of once per tile. */
#define MB200_CONFIG_THROUGHPUT 1
/* Variable-state division (STANDARD / morphological data; the reference's *_Std family:
 * CondLikeDown_Std src/likelihood.c:1920, CondLikeRoot_Std :4496, CondLikeScaler_Std :5547,
 * Likelihood_Std :7359, TiProbs_Std :10066).  Every site pattern has its own number of states
 * (m->nStates[c] <= state_count) and its own transition matrices inside a branch's matrix block
 * (m->tiIndex[c]); mb200_set_pattern_states supplies those tables.  P(t) is built by the engine for
 * the equal-frequency Mk model (unordered characters, SYMPI_EQUAL: pNoChange / pChange per state
 * count and category, src/likelihood.c:10135-10173); the root pass includes the correction for
 * unobservable (dummy) patterns, Likelihood_Std's coding bias (src/likelihood.c:7401-7423, 7537). */
#define MB200_CONFIG_VARIABLE_STATES 2
/* Hint: the reference runs this division on its scalar kernels (SetLikeFunctions picks CondLikeDown_NUC4 / _Gen
 * instead of the SIMD variants when ancestral states or site rates are reported, src/mcmc.c:17971-17992).  The
 * engine's operation order does not depend on it (lnL agrees to rounding either way); a CPU restatement that
 * reproduces the reference bit for bit (oracle/) follows the scalar kernels' order when it is set. */
#define MB200_CONFIG_SCALAR_KERNELS 4

/* evaluation flags */
/* Root integration follows Likelihood_NUC4_{SSE,AVX,FMA}: when the site scaler is
 * below -200 and likeI > 1e-70 the pattern contributes (lnScaler + log(likeI))
 * (src/likelihood.c:6590-6617); without the flag it follows Likelihood_Gen*
 * and contributes log(likeI) alone (src/likelihood.c:5881-5888). */
#define MB200_FLAG_NUC4_PINVAR_QUIRK  1
/* Terminal-branch shortcut of the scalar and *_Gen_SSE kernels (preLikeL/R/A,
 * src/likelihood.c:236-260, 2441-2520): on a tip WITHOUT partially ambiguous patterns a
 * missing/gap observation contributes exactly 1.0 to every ancestral state instead of
 * sum_j P[i][j] (which is 1 only up to rounding).  The 4-state SSE/AVX/FMA kernels treat
 * tips as dense vectors and do not take the shortcut (src/likelihood.c:1121-1250). */
#define MB200_FLAG_TIP_SHORTCUTS      2
/* Float-range guard for callers that rescale sparsely (scale_write on a subset of the nodes: the dynamic scheme of
 * src/mbbeagle.c:429-534).  With the flag set, a rescaler maximum or an unscaled root likelihood below 1e-24 --
 * values whose smaller siblings are on their way out of the float range -- ends the evaluation with
 * MB200_EVAL_UNDERFLOW, so that the caller can repeat it with every node rescaled before precision is lost
 * (without the flag only a dead likelihood, < 1e-300 like the reference, does).  4-state instances, any category
 * count; ignored otherwise. */
#define MB200_FLAG_RANGE_GUARD        4

typedef struct mb200_instance_config
{
    int tip_count;        /* numLocalTaxa; partials buffers 0..tip_count-1 are tips       */
    int partials_count;   /* m->numCondLikes: tips + (chains+1)*nIntNodes                 */
    int state_count;      /* m->numModelStates (2..64)                                    */
    int pattern_count;    /* m->numChars, unique site patterns                            */
    int category_count;   /* m->numRateCats (Gamma) or numOmegaCats; 1..20                */
    int matrix_count;     /* m->numTiProbs: (chains+1)*nNodes                             */
    int scaler_count;     /* m->numScalers: (chains+1)*(nIntNodes+1), node + site scalers */
    int eigen_count;      /* cijk slots: chains+1                                         */
    int weight_rows;      /* rows of numSitesOfPat (1, or numChains when reweighting)     */
    int device;           /* CUDA device ordinal                                          */
    int max_evaluations;  /* largest `count` ever passed to mb200_evaluate (>=1)          */
    int flags;            /* MB200_CONFIG_THROUGHPUT | MB200_CONFIG_VARIABLE_STATES | MB200_CONFIG_CIJK_PARTS(n), or 0 */
} mb200_instance_config;

/* One interior-node update: what CondLikeDown / CondLikeRoot + RemoveNodeScalers +
 * CondLikeScaler do for one node of LaunchLogLikeForDivision's post-order loop
 * (src/likelihood.c:7892-7967).  Seven-int BeagleOperation (src/mbbeagle.c:817-843)
 * widened by the third neighbour of the unrooted interior root. */
typedef struct mb200_operation
{
    int dest;          /* partials buffer written                                          */
    int child1;        /* left child partials buffer (index < tip_count => tip)            */
    int matrix1;       /* transition-matrix buffer of the left branch                      */
    int child2;        /* right child                                                      */
    int matrix2;
    int child3;        /* MB200_NONE, or p->anc of the interior root (CondLikeRoot_*)      */
    int matrix3;       /* MB200_NONE, or the interior root's own branch matrix             */
    int scale_write;   /* node-scaler buffer to write after rescaling, MB200_NONE = keep   */
    int scale_remove;  /* node-scaler buffer subtracted from the site scaler first
                          (RemoveNodeScalers), MB200_NONE = nothing to remove              */
} mb200_operation;

/* One branch whose P(t) must be rebuilt (TiProbs_*).  `length` is the branch
 * length after relaxed-clock substitution (src/likelihood.c:9471-9496). */
typedef struct mb200_matrix_update
{
    int    matrix;     /* transition-matrix buffer written                                 */
    int    eigen;      /* cijk slot read                                                   */
    double length;
} mb200_matrix_update;

/* One LaunchLogLikeForDivision call. */
typedef struct mb200_evaluation
{
    int                         matrix_update_count;
    const mb200_matrix_update  *matrix_updates;
    int                         operation_count;
    const mb200_operation      *operations;      /* post-order (intDownPass)               */
    int                         site_scaler_dst; /* m->siteScalerIndex[chain] after flip    */
    int                         site_scaler_src; /* previous site scaler (CopySiteScalers),
                                                    MB200_NONE = ResetSiteScalers           */
    int                         root_buffer;     /* partials of tree->root->left            */
    int                         weights_row;     /* chainId % numChains                     */
    int                         flags;           /* MB200_FLAG_*                            */
    double                      p_invar;         /* 0 when the model has no pInvar          */
    int                         has_p_invar;     /* m->pInvar != NULL                       */
    /* r_k = GetRate(d,chain) / (1-pInvar) * catRate[k] * correctionFactor
       (src/likelihood.c:9438-9464, 9501) */
    double                      category_rates[MB200_MAX_CATEGORIES];
    /* mixture weights w_k: (1-pInvar)/K for Gamma models (src/likelihood.c:5821-5824),
       omega-category frequencies for NY98 (src/likelihood.c:7000) */
    double                      category_weights[MB200_MAX_CATEGORIES];
    /* stationary frequencies of the model states (covarion-adjusted by the caller,
       src/likelihood.c:5797-5818) */
    double                      state_freqs[MB200_MAX_STATES];
    /* Optional eigensystem travelling with the evaluation instead of living in an eigen slot: a
     * cijk block [lambda_re(S), lambda_im(S), c_ijk(S^3)] for matrix updates whose eigen field is
     * MB200_EIGEN_INLINE.  Used for the models MrBayes keeps no eigensystem for (nst = 1, 2:
     * TiProbs_JukesCantor / _Fels / _Hky closed forms, src/likelihood.c:9289-9960); the seam derives
     * the eigensystem of their rate matrix per evaluation.  4-state models only.  NULL otherwise. */
    const double               *inline_eigen;
} mb200_evaluation;

/* ---- library ---------------------------------------------------------------------- */
int         mb200_abi_version (void);
const char *mb200_version_string (void);
const char *mb200_error_string (int code);
int         mb200_device_count (void);     /* sm_90-class devices visible; 0 = none        */

/* ---- instance ---------------------------------------------------------------------- */
int mb200_create_instance   (const mb200_instance_config *config, int *instance);
int mb200_finalize_instance (int instance);

/* ---- static data ------------------------------------------------------------------- */
/* state_masks[c] bit s set <=> model state s is compatible with the observation at
 * pattern c (missing/gap: all state_count bits set).  Hidden covarion states are
 * replicated by the caller exactly as src/mcmc.c:6402-6411 does. */
int mb200_set_tip_states      (int instance, int tip, const uint64_t *state_masks);
int mb200_set_pattern_weights (int instance, int row, const float *weights);
/* Variable-state instances only (MB200_CONFIG_VARIABLE_STATES), once, before the first evaluation:
 *   state_counts[c]    m->nStates[c], 2 .. state_count                    (src/bayes.h:1331)
 *   matrix_offsets[c]  m->tiIndex[c]: where pattern c's category-0 matrix starts inside a branch's
 *                      block of matrix_length floats; category k follows at + k * nStates^2
 *                      (src/likelihood.c:1958-1961)                        (src/bayes.h:1329)
 *   freq_offsets[c]    m->bsIndex[c]: where pattern c's state frequencies start inside
 *                      mb200_evaluation.state_freqs (freq_offsets[c] + nStates[c] <= 64)   (:1330)
 *   matrix_length      m->tiProbLength: floats per branch (src/mcmc.c:5799-5828)
 *   dummy_patterns     m->numDummyChars: leading all-constant patterns that only feed the
 *                      unobservable-pattern correction (AddDummyChars, src/model.c:176-224)
 *   uncompressed_sites m->numUncompressedChars: sites the correction applies to (:7537)
 * Host layout of partials for these instances is the reference's ragged one: [k][c][nStates[c]]
 * (src/likelihood.c:1941-1943); of a transition-matrix buffer: matrix_length floats. */
int mb200_set_pattern_states (int instance, const int *state_counts, const int *matrix_offsets,
                              const int *freq_offsets, int matrix_length, int dummy_patterns,
                              int uncompressed_sites);

/* ---- eigen systems ----------------------------------------------------------------- */
/* block = [lambda_re(S), lambda_im(S), c_ijk(S*S*S)] exactly as m->cijks[idx] holds it
 * (src/likelihood.c:9467-9468; src/utils.c:9734-9746) */
int mb200_set_cijk (int instance, int eigen, const double *block);
/* row-major V and V^-1 and real eigenvalues; c_ijk = V[i][k]*Vinv[k][j] is formed on
 * the device */
int mb200_set_eigen_decomposition (int instance, int eigen, const double *eigvecs,
                                   const double *inverse_eigvecs, const double *eigvals);
/* The eigensolver itself on the device: replaces the host half of UpDateCijk (GetEigens src/utils.c:11201 +
 * CalcCijk src/utils.c:9734, called at src/likelihood.c:10626-10760).  rate_matrices = the slot's Q matrices
 * as SetNucQMatrix / SetProteinQMatrix fill them (row-major S x S, one per eigen part: category_count of them
 * for instances created with omega categories, else one), already scaled the way UpDateCijk scales them;
 * state_freqs = the stationary frequencies (all > 0) the matrices are reversible with respect to
 * (pi_i q_ij == pi_j q_ji; the caller checks, the solver symmetrises).  Asynchronous: the call returns after
 * queueing the copy and three kernels on the instance's stream; a failure to converge is reported by the next
 * mb200_evaluate / _end as MB200_ERROR_GENERAL.  S <= 64, not for variable-state instances.
 * like_eigen: a slot whose matrices these are a small change of (the chain's current state when a move proposes
 * new kappa / omega / frequencies), or MB200_NONE; when that slot was solved by this call too, its eigenvectors
 * start the iteration (fewer sweeps).  A hint only: the result does not depend on it beyond rounding. */
int mb200_set_rate_matrices (int instance, int eigen, int like_eigen, const double *rate_matrices, const double *state_freqs);

/* ---- node-granular verbs (the function-pointer / BEAGLE-verb level) ---------------- */
int mb200_update_transition_matrices (int instance, const mb200_matrix_update *updates,
                                      int count, const double *category_rates,
                                      const double *state_freqs);
/* site_scaler = cumulative scale buffer that node scalers are removed from / added to
 * (MB200_NONE: leave site scalers alone) */
int mb200_update_partials (int instance, const mb200_operation *operations, int count,
                           int site_scaler);
int mb200_reset_scalers   (int instance, int scaler);                 /* ResetSiteScalers */
int mb200_copy_scalers    (int instance, int dst, int src);           /* CopySiteScalers  */
int mb200_root_log_likelihood (int instance, int root_buffer, int site_scaler,
                               int weights_row, const double *state_freqs,
                               const double *category_weights, int has_p_invar,
                               double p_invar, int flags, double *lnL, int *status);

/* ---- fused, chain-batched evaluation (the hot path) -------------------------------- */
/* count evaluations (normally one per MC^3 chain) in ONE pass: P(t) build, pruning over
 * each evaluation's operation list with the rescaler fused, root integration and the
 * weighted log-sum.  lnL[i] and status[i] are written for every evaluation.
 * The evaluations of one call must not write the same buffers. */
int mb200_evaluate (int instance, const mb200_evaluation *evaluations, int count,
                    double *lnL, int *status);

/* The same call in two halves, so that the divisions (partitions) of one chain -- separate
 * instances, separate streams -- are in flight together and their launch latencies overlap:
 * begin() validates, packs and launches and returns at once; end() waits for the results.
 * One evaluation may be in flight per instance.  This is what the reference's partition-batched
 * accelerator entry does in one BEAGLE call (LaunchBEAGLELogLikeMultiPartition, src/mbbeagle.h:29;
 * LaunchLogLikeForBeagleMultiPartition, src/likelihood.c:7792). */
int mb200_evaluate_begin (int instance, const mb200_evaluation *evaluations, int count);
int mb200_evaluate_end   (int instance, double *lnL, int *status);

/* ---- read-back / seeding (parity tests, debugging) --------------------------------- */
/* host layout of partials: [k][c][s] floats, the reference's scalar layout
 * (src/mcmc.c:5756, 6397-6413) */
int mb200_get_partials          (int instance, int buffer, float *out);
int mb200_set_partials          (int instance, int buffer, const float *in);
int mb200_get_transition_matrix (int instance, int matrix, float *out);  /* [k][i][j]     */
int mb200_set_transition_matrix (int instance, int matrix, const float *in);
int mb200_get_scalers           (int instance, int scaler, float *out);  /* [c]           */
int mb200_set_scalers           (int instance, int scaler, const float *in);

/* ---- device-resident replay (benchmark "value" leg; inputs already in HBM) --------- */
/* Pack evaluations into the engine's device job format and keep them resident; returns a
 * handle.  mb200_replay launches the fused pass for a packed batch without any
 * host<->device copy; results stay on the device until mb200_replay_results. */
int mb200_pack_evaluations (int instance, const mb200_evaluation *evaluations, int count,
                            int *batch);
int mb200_replay           (int instance, int batch);
int mb200_replay_results   (int instance, int batch, double *lnL, int *status);
/* the same launch with the results delivered like mb200_evaluate_begin / _end delivers them (16-byte
 * records written by the kernel into pinned host memory, the caller polls): resident descriptors in,
 * lnL on the host out, no copy and no stream synchronisation.  One launch in flight per instance.
 * Small 4-state batches on an instance that is alone on its device are served by a kernel that stays
 * resident on the instance's stream after mb200_replay_end returns: until the next other call on the
 * instance, mb200_synchronize, or about 100 us without a new mb200_replay_begin. */
int mb200_replay_begin     (int instance, int batch);
int mb200_replay_end       (int instance, double *lnL, int *status);
/* A batch whose replay_begin has not been collected by replay_end yet cannot be freed: the call
 * returns MB200_ERROR_OUT_OF_RANGE, the code replay_begin uses for one evaluation in flight. */
int mb200_free_batch       (int instance, int batch);
int mb200_synchronize      (int instance);
/* the CUDA stream (cudaStream_t as void*) all work of the instance is issued on, so a
 * caller can bracket it with its own events */
int mb200_get_stream       (int instance, void **stream);
/* kernels launched by the instance since creation (bench.py's gpu_launches) */
int mb200_get_launch_count (int instance, long long *launches);
/* the same count per kernel family, so a caller (or a test) can tell WHICH path served it: the
 * 4-state shuffle kernel, the wgmma tensor-core kernel (20 / 61 states), the CUDA-core kernel for
 * any other state count, the variable-state (Std) kernel, stand-alone P(t) builds, set-up kernels */
#define MB200_KERNEL_NUC4     0
#define MB200_KERNEL_TENSOR   1
#define MB200_KERNEL_GENERIC  2
#define MB200_KERNEL_STD      3
#define MB200_KERNEL_TIPROBS  4
#define MB200_KERNEL_SETUP    5
#define MB200_KERNEL_KINDS    6
/* two sub-counts of the 4-state launches, for the same purpose (not added into mb200_get_launch_count): the job
 * read from the kernel's parameter block, and throughput mode's one CTA per evaluation (MB200_CONFIG_THROUGHPUT) */
#define MB200_KERNEL_NUC4_PARAMS    6
#define MB200_KERNEL_NUC4_PER_EVAL  7
#define MB200_KERNEL_COUNTERS       8
int mb200_get_kernel_launches (int instance, int kind, long long *launches);
/* Device-side timing of the dominant (fused pruning) kernel: when enabled, every launch of
 * it is bracketed by CUDA events on the instance's stream.  mb200_get_kernel_time
 * synchronises, returns the summed duration (ms) and the number of launches measured since
 * the last call, and clears the measurements (at most the 2048 most recent launches are kept). */
int mb200_set_kernel_timing (int instance, int enabled);
int mb200_get_kernel_time   (int instance, double *milliseconds, int *launches);

#ifdef __cplusplus
}
#endif
#endif /* MB200_H_ */
