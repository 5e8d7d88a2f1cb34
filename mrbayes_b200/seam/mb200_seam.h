/*
 * mb200_seam.h -- what the seam adds on top of the reference's src/mbbeagle.h.
 *
 * The seam TU (mb200_seam.c) defines the mbbeagle.h entry points
 * (InitBeagleInstance, LaunchBEAGLELogLikeForDivision, TreeTiProbs_Beagle,
 * TreeCondLikes_Beagle_*, TreeLikelihood_Beagle) against the H100 engine; this
 * header declares only the few extra symbols a caller needs.
 */
#ifndef MB200_SEAM_H_
#define MB200_SEAM_H_

#include "mb200.h"

/* Replacement for LaunchLogLikeForDivision (src/likelihood.c:7851): returns YES (1)
 * when the engine evaluated the division (lnL / abortMove set like the reference),
 * NO (0) when the division's model is outside the engine's coverage and the caller
 * must use the reference's own function-pointer path. */
int       MB200LaunchLogLikeForDivision (int chain, int d, MrBFlt *lnL);
int       MB200SeamDivisionSupported (ModelInfo *m);
int       MB200SeamClosedFormModel (ModelInfo *m);     /* nst = 1, 2 4x4 models: eigensystem sent inline */
/* Replacement for the division loop of LogLike (src/mcmc.c:7421-7441): every division of `chain`
 * that needs updating is launched before any result is waited for, so the partitions of a chain
 * overlap on the device.  Divisions outside the engine's coverage go to `cpuPath` (the reference's
 * own LaunchLogLikeForDivision body).  Returns the chain's log likelihood (MRBFLT_NEG_MAX and
 * abortMove = YES on a numerical failure, like the reference). */
MrBFlt    MB200LogLike (int chain, void (*cpuPath) (int chain, int d, MrBFlt *lnL));
/* Chain-batched generations (RunChain's chain loop cut in two around LogLike, src/mcmc.c:16718-16938; see
 * mb200_seam.c and INTEGRATION.md): all local chains' evaluations of a generation in ONE device call. */
void      MB200BatchEnable (int enable);
int       MB200BatchBegin (void);
void      MB200BatchEnterChain (int chain, int phase);
void      MB200BatchLeaveChain (int chain, int phase);
void      MB200BatchQueueLogLike (int chain);
void      MB200BatchFlush (void);
MrBFlt    MB200BatchFinishLogLike (int chain);
void      MB200SeamFinalize (void);
/* CUDA device a division's buffers live on (local rank, MB200_DEVICE, MB200_SHARD=partitions) */
int       MB200SeamDeviceFor (int division);
/* the engine instance a division needs (what InitBeagleInstance creates) */
void      MB200SeamDivisionConfig (ModelInfo *m, int division, mb200_instance_config *cfg);

/* Node-granular function-pointer forms (typedefs src/bayes.h:960-965): same signatures as the
 * reference's TiProbs_*, CondLikeDown_*, CondLikeRoot_*, CondLikeScaler_*, Likelihood_* families
 * (src/likelihood.h:43-162), installable by SetLikeFunctions (src/mcmc.c:17918).  They record the
 * evaluation while the reference's own LaunchLogLikeForDivision loop runs and launch it as one fused
 * pass from Likelihood_B200.  MB200InstallLikeFunctions points a division's ModelInfo at them. */
int       TiProbs_B200        (TreeNode *p, int division, int chain);
int       CondLikeDown_B200   (TreeNode *p, int division, int chain);
int       CondLikeRoot_B200   (TreeNode *p, int division, int chain);
int       CondLikeScaler_B200 (TreeNode *p, int division, int chain);
int       Likelihood_B200     (TreeNode *p, int division, int chain, MrBFlt *lnL, int whichSitePats);
int       MB200InstallLikeFunctions (int division);
/* Host readers of conditional-likelihood buffers (SURVEY 8f4): CondLikeUp_* (src/likelihood.c:4574-4925),
 * PrintAncStates_* (src/mcmc.c:10713, 10902), PrintSiteRates_Gen (src/mcmc.c:12212) run on the HOST arrays m->condLikes /
 * m->tiProbs / m->scalers at sample time (src/mcmc.c:13029, 13141, 13151).  MB200InstallReaders wraps the three function
 * pointers of a division: before the reference's own reader runs, the cold chain's current buffers are copied from the
 * device into those arrays (once per evaluation state).  Returns ERROR when the division needs no readers or the backend
 * has no read-back. */
int       CondLikeUp_B200     (TreeNode *p, int division, int chain);
int       PrintAncStates_B200 (TreeNode *p, int division, int chain);
int       PrintSiteRates_B200 (TreeNode *p, int division, int chain);
int       MB200InstallReaders (int division);
int       PosSelProbs_B200 (TreeNode *p, int division, int chain);     /* report possel=yes   */
int       SiteOmegas_B200 (TreeNode *p, int division, int chain);      /* report siteomega=yes */
long long MB200SeamUpdateCount (int division);   /* node*pattern*rate CL updates issued  */
void      MB200SeamCijkTimes (double *secHost, double *secUpload, long long *updates);   /* eigensystem work on the host */
long long MB200SeamDeviceEigens (void);          /* MB200_EIGEN=device: eigensystems computed by the backend */
long long MB200SeamRescaleRetries (void);        /* MB200_RESCALE=dynamic: evaluations repeated after an underflow */
int       MB200SeamInstance (int division);      /* engine instance of a division, or -1 */

/* Every engine call the seam makes goes through this table, so a test harness can
 * record the calls (golden vectors), shadow them, or both. */
typedef struct
    {
    int (*create_instance)     (const mb200_instance_config *config, int *instance);
    int (*finalize_instance)   (int instance);
    int (*set_tip_states)      (int instance, int tip, const uint64_t *state_masks);
    int (*set_pattern_weights) (int instance, int row, const float *weights);
    int (*set_cijk)            (int instance, int eigen, const double *block);
    int (*evaluate)            (int instance, const mb200_evaluation *evaluations, int count,
                                double *lnL, int *status);
    /* optional (may be NULL: the seam then evaluates synchronously) */
    int (*evaluate_begin)      (int instance, const mb200_evaluation *evaluations, int count);
    int (*evaluate_end)        (int instance, double *lnL, int *status);
    /* variable-state (STANDARD data) divisions; NULL: those divisions stay on the reference's kernels */
    int (*set_pattern_states)  (int instance, const int *state_counts, const int *matrix_offsets,
                                const int *freq_offsets, int matrix_length, int dummy_patterns,
                                int uncompressed_sites);
    /* optional read-back (host readers of conditional-likelihood buffers, MB200InstallReaders); NULL: divisions
       that report ancestral states / site rates stay on the reference's kernels */
    int (*get_partials)          (int instance, int buffer, float *out);
    int (*get_transition_matrix) (int instance, int matrix, float *out);
    int (*get_scalers)           (int instance, int scaler, float *out);
    /* optional: a transition-matrix buffer filled by the caller (STANDARD-data divisions whose matrices the reference's own
       TiProbs_Std builds on the host: ordered characters, unequal state frequencies); NULL: those divisions stay on the
       reference's kernels */
    int (*set_transition_matrix) (int instance, int matrix, const float *in);
    /* optional: eigensystems computed by the backend from the rate matrices (MB200_EIGEN=device); NULL: the host's
       UpDateCijk computes them and set_cijk ships the block */
    int (*set_rate_matrices)     (int instance, int eigen, int like_eigen, const double *rate_matrices, const double *state_freqs);
    } MB200SeamBackend;

void      MB200SeamSetBackend (const MB200SeamBackend *backend);   /* NULL = the engine  */

#endif /* MB200_SEAM_H_ */
