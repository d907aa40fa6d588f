/* pb_bss_b200 C ABI -- the drop-in boundary of the pb_bss EM / beamforming hot path.
 *
 * pb_bss (the reference) is a pure NumPy library; its only native seam is the
 * import-time hook around two Cython LAPACK loops
 * (pb_bss/extraction/beamformer.py:38-56 ->
 *  pb_bss/extraction/cythonized/get_gev_vector.pyx:42,
 *  pb_bss/extraction/cythonized/c_eig.pyx:14).  This library moves the whole
 * per-bin hot path behind one C ABI; each entry point names the reference
 * function(s) it replaces.  A maintainer binds it with ctypes exactly like
 * pb_bss_b200/_lib.py does (see INTEGRATION.md).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer owned by the caller and the library never frees
 *    caller memory (pbb_cacgmm_fit additionally accepts PINNED host pointers, see there).
 *    The library itself owns three small things per device, created on first use and kept
 *    for the life of the process: a non-blocking side stream with two events (streamed
 *    upload of pbb_cacgmm_fit), a cache of at most 16 task-order tables (4 bytes per task,
 *    streamed upload only) and the occupancy numbers of its persistent kernels;
 *  - `stream` is a cudaStream_t passed as void*; all work is stream-ordered
 *    and asynchronous, no entry synchronises the device or the stream;
 *  - limits: D < 35, K < 20 (the reference asserts the same, cacgmm.py:197,249-250);
 *    pbb_streamed_task_order packs the bin into 16 bits (F <= 65535; pbb_cacgmm_fit only uses
 *    such a table for F <= 4096 and schedules larger problems without it);
 *  - thread safety: entries may be called concurrently from several host threads on
 *    different streams.  pbb_last_error() is thread-local.  Two streamed fits (pinned-host
 *    input) on the SAME device are serialised while they enqueue, because they share the
 *    side stream; everything else only reads library state;
 *  - return value: 0 = ok, -i = argument i (1-based) invalid (LAPACK INFO<0
 *    convention, cf. get_gev_vector.pyx:130-147), > 0 = CUDA runtime error
 *    code; pbb_last_error() gives the message (thread-local);
 *  - numerical failures (non-finite covariance, not-positive-definite noise
 *    PSD, ...) are reported through a caller-provided device status word
 *    `int* status` (0 = ok, else 1 + index of the first failing matrix/bin),
 *    which the caller reads after synchronising -- the reference raises
 *    AssertionError / ValueError at the same places;
 *  - all arithmetic is IEEE fp64; `dtype` only selects the STORAGE type of the
 *    complex observation (PBB_C64 = float2, PBB_C128 = double2).
 */
#ifndef PBB_H_
#define PBB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PBB_C64 0
#define PBB_C128 1

/* covariance_norm of CACGMMTrainer.fit (pb_bss/distribution/cacgmm.py:152) */
#define PBB_NORM_NONE 0       /* covariance_norm=False */
#define PBB_NORM_EIGENVALUE 1 /* 'eigenvalue' (default) */
#define PBB_NORM_TRACE 2      /* 'trace' */

/* weight_constant_axis (pb_bss/distribution/mixture_model_utils.py:133-203) */
#define PBB_WEIGHT_TIME 0     /* (-1,): one weight per (bin, class) */
#define PBB_WEIGHT_CONST 1    /* -2: constant 1/K */
#define PBB_WEIGHT_TIED_TIME 2 /* (-3,): frequency-tied weights, one per (class, frame): array (K, T) */
#define PBB_WEIGHT_TIED 3     /* (-3, -1): frequency-tied, one per class: array (K) */
#define PBB_WEIGHT_FRAME 4    /* one weight per (bin, frame), the same for every class: array (F, T); only
                                 pbb_log_pdf_to_affiliation (GMM / VMFMM weight_constant_axis (-2,)) */
#define PBB_WEIGHT_BCAST 8    /* PBB_WEIGHT_BCAST | 1 (spans F) | 2 (spans K) | 4 (spans T): a contiguous (F', K', T')
                                 array with F' = F or 1 etc., read with stride 0 along the dims whose bit is clear,
                                 i.e. any weight that broadcasts to (F, K, T); only pbb_log_pdf_to_affiliation */

const char* pbb_last_error(void);
int pbb_version(void);

/* Launch accounting and optional CUDA-event timing of the library's own kernels
 * (used by bench.py for `gpu_launches` and the roofline of the dominant kernel).
 * pbb_launch_count: the kernel launches so far; each launch also gets its own profile record. */
long long pbb_launch_count(void);
void pbb_profile_enable(int on);
void pbb_profile_reset(void);
/* Sums the recorded launches per kernel, returns the kernel with the largest
 * total device time (ms) and its launch count, and clears the records.
 * Synchronises on the recorded events.  Return value: number of distinct kernels. */
int pbb_profile_dominant(char* name, int name_len, double* total_ms, int* launches);
void pbb_profile_dump(void); /* every recorded launch to stderr */

/* ------------------------------------------------------------------------
 * Observation normalisation.
 * swap=1: pb_bss/distribution/complex_angular_central_gaussian.py:34-55
 *         (unit norm over D, zero vectors stay zero, output (F, D, T));
 * swap=0: pb_bss/distribution/complex_watson.py:16-29 (output (F, T, D)).
 * y: (F, T, D) complex of `dtype`; z: same dtype. */
int pbb_normalize_observation(const void* y, void* z, int F, int T, int D,
                              int dtype, int swap, void* stream);

/* ------------------------------------------------------------------------
 * cACGMM (pb_bss/distribution/cacgmm.py).
 *
 * Device model of one fit: for every (bin f, class k)
 *   eigenvectors (F, K, D, D) complex128 row-major, column e = e-th vector
 *   eigenvalues  (F, K, D)    float64, ascending
 *   weight       (F, K)       float64
 * = CACGMM.weight / cacg.covariance_eigenvectors / covariance_eigenvalues
 * (cacgmm.py:58-62, complex_angular_central_gaussian.py:78-79).
 */
typedef struct pbb_cacgmm_options {
  int iterations;          /* > 0 */
  int covariance_norm;     /* PBB_NORM_* */
  int weight_mode;         /* PBB_WEIGHT_* */
  int hermitize;           /* accepted for API parity; the scatter matrix is
                              accumulated in Hermitian form either way */
  double affiliation_eps;  /* clip of the posterior, cacgmm.py:154 */
  double eigenvalue_floor; /* cacgmm.py:155 */
  int frames_per_block;    /* 0 = library default; tuning knob */
  int reserved;            /* bit 0: force the multi-kernel (non-persistent) path;
                              every other bit must be 0 */
} pbb_cacgmm_options;

/* Host-only helper (no GPU needed): the task order pbb_cacgmm_fit uses for a streamed upload.
 * order (HOST, F * iterations ints): order[ticket] = bin | iteration << 16.  `arrive` bins join
 * per time slot, at most `cap` tasks run per slot; every (bin, it) comes after (bin, it - 1). */
int pbb_streamed_task_order(int F, int iterations, int arrive, int cap, int* order);

/* Host only: which persistent kernel pbb_cacgmm_fit runs for a problem on a GPU with `sms` SMs, and how one EM
 * iteration of a bin is split (DESIGN.md 6.1).  lean = no saliency / activity mask / user-supplied model and
 * eigenvalue_floor in the product-softmax range; streamed = pinned host input (streamed upload).
 * *kernel: 0 = em_ws_kernel (task kernel, lean D = 8), 1 = em_sticky_kernel (one cluster of *split CTAs per bin for
 * the whole fit), 2 = em_persistent_kernel (lean D = 4 / 6, full variant); *split = parts per bin-iteration (1 =
 * none).  This is the function the fit itself uses, except that the sticky kernel's clusters are modelled as two CTAs
 * per SM placed anywhere; pbb_cacgmm_fit instead asks the device how many clusters it runs at once, which on a GPU
 * with uneven GPCs can pick a smaller cluster.  The complex Watson fit (pbb_cwmm_fit) always runs
 * em_persistent_kernel, split as reported for lean = 1, streamed = 1. */
int pbb_em_dispatch(int F, int T, int D, int K, int lean, int streamed, int sms, int* kernel, int* split);

/* Host only: the plan of the last persistent fit (pbb_cacgmm_fit / pbb_cwmm_fit) the calling host thread launched.
 * *kernel and *split as in pbb_em_dispatch (*kernel = -1: none yet);
 * *variant: 0 = lean (product-form softmax), 1 = full with the integer-power softmax, 2 = full with the log-domain
 * softmax, 3 = complex Watson. */
int pbb_em_last_plan(int* kernel, int* split, int* variant);

/* Bytes of scratch pbb_cacgmm_fit / _predict need for this problem size. */
size_t pbb_cacgmm_workspace_bytes(int F, int T, int D, int K);

/* CACGMMTrainer.fit (cacgmm.py:142-280): full EM loop on the device.
 *  y            (F, T, D) complex `dtype`, un-normalised STFT
 *  init_aff     (F, K, T) float64 initial affiliations, or NULL for a warm
 *               start from the model already stored in
 *               eigenvectors/eigenvalues/weight (cacgmm.py:229-234)
 *  saliency     (F, T) float64 or NULL
 *  activity     (F, K, T) uint8 source_activity_mask or NULL
 *  outputs      eigenvectors, eigenvalues, weight as described above
 *  status       device int, see header comment
 * Host buffers: y, init_aff and the three outputs may also be PINNED
 * (page-locked, mapped) host memory; the kernels then read / write them in place
 * over PCIe.  With y pinned and init_aff given, a small loader kernel on an
 * internal side stream streams the bins in while the EM kernel already iterates
 * on the bins that have arrived (task order: see em_persistent.cuh; the order
 * table, 4 bytes per task, lives in a small library-owned device cache).  The
 * call stays asynchronous with respect to `stream`.
 */
int pbb_cacgmm_fit(const void* y, int dtype, int F, int T, int D, int K,
                   const double* init_aff, const double* saliency,
                   const uint8_t* activity, const pbb_cacgmm_options* opt,
                   void* eigenvectors, double* eigenvalues, double* weight,
                   void* workspace, size_t workspace_bytes, int* status,
                   void* stream);

/* CACGMM.predict / _predict / log_likelihood (cacgmm.py:64-138): one E-step.
 *  affiliation  (F, K, T) float64 out (may be NULL)
 *  quadratic    (F, K, T) float64 out (may be NULL)
 *  loglik       (F) float64 out, per-bin sum_t logsumexp_k log_pdf (may be NULL)
 *  affiliation_eps: 0 for predict (cacgmm.py:73)
 *  weight / weight_mode: (F, K) for PBB_WEIGHT_TIME, ignored for _CONST, (K, T) for
 *  _TIED_TIME and (K) for _TIED (frequency-tied weights, mixture_model_utils.py:187-190)
 */
int pbb_cacgmm_predict(const void* y, int dtype, int F, int T, int D, int K,
                       const void* eigenvectors, const double* eigenvalues,
                       const double* weight, int weight_mode,
                       const uint8_t* activity, double affiliation_eps,
                       double* affiliation, double* quadratic, double* loglik,
                       void* workspace, size_t workspace_bytes, int* status,
                       void* stream);

/* One M-step from given affiliations and quadratic forms:
 * CACGMMTrainer._m_step (cacgmm.py:315-345) =
 * estimate_mixture_weight + ComplexAngularCentralGaussianTrainer._fit
 * (complex_angular_central_gaussian.py:253-342) + from_covariance (:81-132).
 *  quadratic may be NULL (= ones, the first iteration, cacgmm.py:210). */
int pbb_cacgmm_mstep(const void* y, int dtype, int F, int T, int D, int K,
                     const double* affiliation, const double* quadratic,
                     const double* saliency, const pbb_cacgmm_options* opt,
                     void* eigenvectors, double* eigenvalues, double* weight,
                     void* workspace, size_t workspace_bytes, int* status,
                     void* stream);

/* ---- Backward passes of the cACGMM (torch.autograd in pb_bss_b200.distribution.cacgmm).  Conventions as for the
 * beamforming chain below: grad z = dL/dRe z + i dL/dIm z for a real loss L, <A, B> = sum conj(A_ij) B_ij, fp64,
 * fixed-order sums and no atomics (repeated calls are bitwise identical), no status word, enqueue only.  Gradients
 * are written as complex128 / float64; shapes and limits are those of the forward (D < 35, K < 20, any T).
 *
 * Notation: z_t = y_t / |y_t| (a zero frame stays zero), s_t the saliency (1 without), tiny = DBL_MIN.
 * M-step (pbb_cacgmm_mstep):
 *   g_kt = gamma_kt s_t,  S_k = sum_t g_kt,  c_kt = g_kt / max(q_kt, 10 tiny),  Psi_k = sum_t c_kt z_t z_t^H,
 *   C_k = D Psi_k / max(S_k, tiny);  'trace': C'_k = C_k / max(tr C_k, tiny), otherwise C'_k = C_k;
 *   C'_k = V diag(mu) V^H;  'eigenvalue': lam_i = max(mu_i / max(mu_max, tiny), floor), else lam_i = max(mu_i,
 *   mu_max floor);  w_k = S_k / T (no saliency), S_k / sum_j |S_j| (saliency; a zero sum counts as 1e-10), 1 / K (-2).
 * E-step (pbb_cacgmm_predict), with B^-1 = V diag(1 / lam) V^H and ld = sum log lam:
 *   q_kt = max(|z_t^H B_k^-1 z_t|, tiny),  lp_kt = -D log q_kt - ld_k,  a_kt = exp(lp_kt - max_j lp_jt) w_k act_kt,
 *   gamma_kt = clip(a_kt / max(sum_j a_jt, tiny), eps, 1 - eps) (no clip for eps = 0),
 *   loglik_f = sum_t logsumexp_k lp_kt (without the weights).
 * Backward of the E-step, per frame (gb = grad gamma where the clip is not active, else 0):
 *   abar_k = (gb_k - sum_j gb_j gamma_j) / den (den = sum_j a_j > tiny; gb_k / tiny otherwise),
 *   lpbar_k = abar_k w_k act_k e_k + grad_loglik e_k / sum_j e_j (e_k = exp(lp_k - max lp)),
 *   qbar_k = grad_q_k - D lpbar_k / q_k,  qbar_raw_k = qbar_k sign(z^H B_k^-1 z) where q_k > tiny, else 0;
 *   grad z = sum_k 2 qbar_raw_k B_k^-1 z,  Bbar_k = sum_t qbar_raw_kt z_t z_t^H,  ldbar_k = -sum_t lpbar_kt,
 *   grad V_k = 2 Bbar_k V_k diag(1 / lam),  grad lam_ki = -v_i^H Bbar_k v_i / lam_i^2 + ldbar_k / lam_i,
 *   grad w_k = sum_t abar_kt e_kt act_kt.
 * Backward of the M-step, per (bin, class), from V (the forward's output) and the raw eigenvalues
 * mu_i = v_i^H C' v_i of the recomputed scatter (no second eigensolve):
 *   mubar_i = lambar_i / m (pass_i), plus, on the top eigenvector (the forward's last), -sum_i pass_i lambar_i mu_i / m^2
 *   while mu_max > tiny ('eigenvalue', m = max(mu_max, tiny), pass_i: lam_i > floor); mubar_i = lambar_i (pass_i) and
 *   floor lambar_i onto the top otherwise (pass_i: lam_i > lam_max floor).  The floors pass no gradient.
 *   M_ii = mubar_i; M_ij = G_ij / (mu_j - mu_i) with G = V^H Vbar, except where |mu_j - mu_i| <= 2^-26 mu_max (a tie):
 *   there M_ij = -lam' (G_ij + conj G_ji) / (2 (lam_i + lam_j)) if neither eigenvalue is floored (lam' = d lam / d mu:
 *   1 / m for 'eigenvalue', else 1), the Daleckii-Krein limit -lam' P_ij / lam^2 of a B^-1 consumer, whose
 *   G = 2 P diag(1 / lam) with P = V^H Bbar V.  Every pair of floored eigenvalues gives 0 (1 / lam is constant on the
 *   floor), so a rank-deficient scatter gives finite gradients; a floored and an unfloored eigenvalue take the divided
 *   difference, but 0 where |mu_j - mu_i| <= 64 u D mu_max (both at the floor's kink, within the rounding of mu).  Cbar' = V (M + M^H) / 2 V^H.  This is
 *   exact for every loss that sees the model through B^-1 and ld only (E-step, predict, log_likelihood); for a loss on
 *   V itself it is the gradient with the phase held fixed, and at a tie a convention.  At a tied top eigenvalue m is
 *   the Rayleigh quotient of the forward's last eigenvector, held fixed.
 *   'trace': Cbar = Cbar' / tau - Re<Cbar', C'> / tau I (tau = tr C > tiny; Cbar' / tiny otherwise).
 *   Psibar_k = D Cbar_k / S_k,  Sbar_k = -Re<Cbar_k, C_k> / S_k + the weight's share (wbar_k / T, or
 *   wbar_k / n - sum_j wbar_j S_j / n^2 with n = sum_j |S_j|); a class with S_k <= tiny passes no gradient (the
 *   forward forms its covariance as D Psi_k / tiny, a finite model: C_k = 0 at S_k = 0);
 *   cbar_kt = z_t^H Psibar_k z_t,  grad z_t = sum_k 2 c_kt Psibar_k z_t,  gbar_kt = cbar_kt / max(q_kt, 10 tiny) + Sbar_k,
 *   grad gamma_kt = gbar_kt s_t,  grad q_kt = -cbar_kt g_kt / q_kt^2 (q_kt > 10 tiny, else 0),
 *   grad s_t = sum_k gbar_kt gamma_kt.
 * Both: grad y_t = (grad z_t - z_t Re(z_t^H grad z_t)) / |y_t|, zero for an all-zero frame.  A bin with a zero model
 * eigenvalue (eigenvalue_floor = 0) or a non-finite sample gets NaN gradients in that bin only. */
size_t pbb_cacgmm_predict_backward_workspace_bytes(int F, int T, int D, int K);

/* Differentiates pbb_cacgmm_predict with a per-bin weight (F, K) (PBB_WEIGHT_TIME; pass 1 / K for _CONST).
 * affiliation / quadratic: the forward's outputs (F, K, T), so the forward's softmax variant does not matter;
 * grad_affiliation, grad_quadratic (F, K, T) and grad_loglik (F) may each be NULL (zero).  Writes grad_y (F, T, D)
 * complex128, grad_eigenvectors (F, K, D, D) complex128, grad_eigenvalues (F, K, D) and grad_weight (F, K). */
int pbb_cacgmm_predict_backward(const void* y, int dtype, int F, int T, int D, int K,
                                const void* eigenvectors, const double* eigenvalues, const double* weight,
                                const uint8_t* activity, double affiliation_eps,
                                const double* affiliation, const double* quadratic,
                                const double* grad_affiliation, const double* grad_quadratic,
                                const double* grad_loglik, void* grad_y, void* grad_eigenvectors,
                                double* grad_eigenvalues, double* grad_weight, void* workspace,
                                size_t workspace_bytes, void* stream);

size_t pbb_cacgmm_mstep_backward_workspace_bytes(int F, int T, int D, int K);

/* Differentiates pbb_cacgmm_mstep (opt: the forward's options, weight_mode PBB_WEIGHT_TIME or _CONST).
 * eigenvectors / eigenvalues: the forward's outputs; grad_eigenvectors (F, K, D, D), grad_eigenvalues (F, K, D) and
 * grad_weight (F, K) may each be NULL (zero).  Writes grad_y (F, T, D) complex128, grad_affiliation (F, K, T),
 * grad_quadratic (F, K, T; NULL iff quadratic is NULL) and grad_saliency (F, T; NULL iff saliency is NULL). */
int pbb_cacgmm_mstep_backward(const void* y, int dtype, int F, int T, int D, int K,
                              const double* affiliation, const double* quadratic, const double* saliency,
                              const pbb_cacgmm_options* opt, const void* eigenvectors,
                              const double* eigenvalues, const void* grad_eigenvectors,
                              const double* grad_eigenvalues, const double* grad_weight, void* grad_y,
                              double* grad_affiliation, double* grad_quadratic, double* grad_saliency,
                              void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Integrated spatial + spectral model (pb_bss/distribution/gcacgmm.py): cACG of the observation combined with a
 * Gaussian over per-(bin, frame) embeddings (F, T, E).  The spatial part reuses pbb_cacgmm_predict (quadratic form)
 * and pbb_cacgmm_mstep; these entries are the pieces around them.  The mixture weights are pbb_axis_sum and
 * pbb_unit_norm.
 * ------------------------------------------------------------------------ */

/* ComplexAngularCentralGaussian._log_pdf (cacg.py:198-201) from the quadratic form: log_pdf = -D log max(|q|, tiny)
 * - sum_d log eigenvalues.  quadratic, log_pdf (F, K, T); eigenvalues (F, K, D). */
int pbb_cacg_log_pdf(const double* quadratic, const double* eigenvalues, int F, int K,
                     int T, int D, double* log_pdf, void* stream);

/* DiagonalGaussian / SphericalGaussian.log_pdf (gaussian.py:57-135) of every embedding under every class:
 * embedding (F, T, E), mean / precision_cholesky (K, E) (spherical: the scalar repeated E times), log_det (K)
 * -> log_pdf (F, K, T).  E <= 64.  diagonal != 0 evaluates the reference's DiagonalGaussian expression, whose einsum
 * '...dD,...nD->...nd' (gaussian.py:79-87) contracts precision_cholesky[d][:] of EVERY class d with the centred
 * observation and sums the squares over d -- reproduced as is, because the model is a drop-in.  diagonal == 2:
 * VonMisesFisher.log_pdf (von_mises_fisher.py:66-81) for the vMF + cACG model: precision_cholesky[k][0] carries the
 * concentration, log_det[k] the log normaliser; out = concentration <mean, x / max(||x||, tiny)> - log_norm. */
int pbb_gaussian_log_pdf(const double* embedding, const double* mean,
                         const double* precision_cholesky, const double* log_det,
                         int F, int T, int E, int K, int diagonal, double* log_pdf,
                         void* stream);

/* GaussianTrainer._fit (gaussian.py:155-193) over the F*T embeddings with weights weight (F, K, T): mean (K, E),
 * covariance (K, E) ('diagonal') or (K) ('spherical'); two passes (mean, then centred second moments), fixed
 * summation order.  scratch: pbb_gaussian_fit_scratch_doubles doubles. */
size_t pbb_gaussian_fit_scratch_doubles(int F, int E, int K);
int pbb_gaussian_fit(const double* embedding, const double* weight, int F, int T, int E,
                     int K, int spherical, double* mean, double* covariance,
                     double* scratch, void* stream);

/* log_pdf_to_affiliation (mixture_model_utils.py:7-55) of scale_a * log_pdf_a + scale_b * log_pdf_b (log_pdf_b may be
 * null) with the weight layouts of pbb_cacgmm_predict; inline_pa != 0:
 * log_pdf_to_affiliation_for_integration_models_with_inline_pa (:58-130) -- per bin the classes of log_pdf_a are
 * re-paired with those of log_pdf_b by the first permutation (itertools order) that maximises the auxiliary function;
 * permutation (F, K) int32 (may be null) receives the choice.  K <= 6.  weight_mode: PBB_WEIGHT_TIME, _CONST, _TIED_TIME,
 * _TIED, _FRAME, or PBB_WEIGHT_BCAST with its bits (the weight of the public
 * log_pdf_to_affiliation_for_integration_models_with_inline_pa, any shape that broadcasts to (F, K, T)). */
int pbb_log_pdf_to_affiliation(const double* log_pdf_a, const double* log_pdf_b,
                               double scale_a, double scale_b, const double* weight,
                               int weight_mode, const uint8_t* activity,
                               double affiliation_eps, int inline_pa, int F, int K, int T,
                               double* affiliation, int* permutation, void* stream);

/* ------------------------------------------------------------------------
 * Embedding mixture models with independent leading dims (pb_bss/distribution/gmm.py, vmfmm.py): B independent
 * models of K classes over N embeddings of dimension E each.  embedding (B, N, E), weights / log pdfs (B, K, N).
 * E <= 64, K <= 6 (the posterior, pbb_log_pdf_to_affiliation with F = B, T = N).  The mixture weights are
 * pbb_axis_sum and pbb_unit_norm. */

/* Gaussian.log_pdf (gaussian.py:36-56) with full covariance: mean (B, K, E), precision_cholesky U (B, K, E, E) (only
 * the upper triangle is read), log_det (B, K) -> log_pdf (B, K, N).  The reference contracts sklearn's
 * upper-triangular precision Cholesky factor with the einsum '...dD,...nD->...nd', i.e. white = U d, where sklearn's
 * own density uses U^T d; the quadratic form is therefore d^T U^T U d and not d^T Sigma^-1 d (they agree for a
 * diagonal Sigma only).  A drop-in returns what the reference returns, so this evaluates U d. */
int pbb_gaussian_full_log_pdf(const double* embedding, const double* mean, const double* precision_cholesky,
                              const double* log_det, int B, int N, int E, int K, double* log_pdf, void* stream);

/* GaussianTrainer._fit (gaussian.py:152-193), covariance_type 'full', per (b, k) with the weights weight (B, K, N):
 * mean (B, K, E) = sum w x / max(sum w, tiny), covariance (B, K, E, E) = sum w (x - mean)(x - mean)^T / that
 * denominator.  Two passes; the N axis is split into chunks whose partial sums are added in chunk order (the chunking
 * depends on B, N, K only), so results are bit-reproducible.  scratch: pbb_gaussian_full_fit_scratch_doubles. */
size_t pbb_gaussian_full_fit_scratch_doubles(int B, int N, int E, int K);
int pbb_gaussian_full_fit(const double* embedding, const double* weight, int B, int N, int E, int K, double* mean,
                          double* covariance, double* scratch, void* stream);

/* sklearn's _compute_precision_cholesky(covariance, 'full') and _compute_log_det_cholesky (Gaussian.__post_init__,
 * gaussian.py:26-34) for M matrices covariance (M, E, E) (lower triangle read): L = cholesky(Sigma),
 * precision_cholesky = (L^-1)^T (M, E, E), log_det = sum log diag (M).  *status (reset by the call) = 1 + index of the
 * first matrix that is not positive definite (sklearn raises ValueError there). */
int pbb_precision_cholesky(const double* covariance, int M, int E, double* precision_cholesky, double* log_det,
                           int* status, void* stream);

/* VonMisesFisher.log_pdf (von_mises_fisher.py:65-79): mean (B, K, E), concentration / log_norm (B, K) ->
 * log_pdf (B, K, N) = concentration <mean, x / max(||x||, tiny)> - log_norm. */
int pbb_vmf_log_pdf(const double* embedding, const double* mean, const double* concentration, const double* log_norm,
                    int B, int N, int E, int K, double* log_pdf, void* stream);

/* The sums of VonMisesFisherTrainer._fit (von_mises_fisher.py:122-137) over x / max(||x||, tiny): resultant (B, K, E)
 * = sum_n w x, total (B, K) = sum_n w; the rest (B*K*E numbers, scipy's ive) is host math.  Same chunked fixed-order
 * reduction and scratch size as pbb_gaussian_full_fit. */
int pbb_vmf_resultant(const double* embedding, const double* weight, int B, int N, int E, int K, double* resultant,
                      double* total, double* scratch, void* stream);

/* ------------------------------------------------------------------------
 * Complex Watson mixture model (pb_bss/distribution/cwmm.py, complex_watson.py).
 *
 * Device model: mode (F, K, D) complex128, concentration (F, K), weight (F, K)
 * = CWMM.weight / complex_watson.mode / .concentration (cwmm.py:21-24).
 * The inverse hypergeometric ratio is the quadratic B-spline of
 * ComplexWatsonTrainer.spline (complex_watson.py:237-256); the caller builds
 * it once with the reference's recipe and passes its knots spline_t[n + 3]
 * and coefficients spline_c[n] (device pointers); it is model state, like the
 * reference's cached_property. */
size_t pbb_cwmm_workspace_bytes(int F, int T, int D, int K);

/* CWMMTrainer.fit / _fit / _m_step (cwmm.py:76-240), affiliation_eps = 0.
 * init_aff (F, K, T) is required (cwmm.py:121-127 draws it on the host). */
int pbb_cwmm_fit(const void* y, int dtype, int F, int T, int D, int K,
                 const double* init_aff, const double* saliency,
                 int iterations, int weight_mode, const double* spline_t,
                 const double* spline_c, int spline_n,
                 double max_concentration, void* mode, double* concentration,
                 double* weight, void* workspace, size_t workspace_bytes,
                 int* status, void* stream);

/* CWMM.predict (cwmm.py:26-52): affiliation (F, K, T) out.  weight: (F, K) for
 * PBB_WEIGHT_TIME, ignored (1/K) for PBB_WEIGHT_CONST, (K, T) / (K) for the
 * frequency-tied PBB_WEIGHT_TIED_TIME / PBB_WEIGHT_TIED (weight_constant_axis (-3,) / (-3, -1)). */
int pbb_cwmm_predict(const void* y, int dtype, int F, int T, int D, int K,
                     const void* mode, const double* concentration,
                     const double* weight, int weight_mode, double* affiliation,
                     void* workspace, size_t workspace_bytes, int* status,
                     void* stream);

/* ------------------------------------------------------------------------
 * Complex Bingham mixture model (pb_bss/distribution/cbmm.py, complex_bingham.py).
 *
 * Device model: eigenvectors (F, K, D, D) complex128 (columns, ascending scatter
 * eigenvalues, like np.linalg.eigh), eigenvalues (F, K, D) = the Bingham parameters
 * lambda (largest 0), weight (F, K) = CBMM.weight / complex_bingham.covariance_eigenvectors /
 * .covariance_eigenvalues.  D is limited to 2..6, the reference's domain
 * (complex_bingham_utils.py:342-348; D = 7 raises KeyError there).
 *
 * Normaliser c(lambda) = 2 pi^D exp[lambda_1..lambda_D], the divided difference of exp
 * (complex_bingham.py:153-164), evaluated as an entry of exp() of the bidiagonal Opitz
 * matrix by scaling and squaring; the E-step first applies the reference's gap rule
 * (sorted neighbours at least 1e-8 apart, :167-203, norm()'s default eps).
 *
 * Parameter solve (find_eigenvalues_v3, :304-425): grad log c(lambda) = s in the differences
 * of neighbouring sorted lambda, bounds [-max_concentration, -1e-8], start -diff(-1 / s),
 * by projected Gauss-Newton with the analytic Jacobian, to max |residual| <= 1e-12 (or until
 * the residual stops decreasing in fp64).  The reference's scipy least_squares stops at
 * residuals of ~1e-7, so its lambda differ from these by up to ~2e-4 relative.
 *
 * Status word (int, 0 = ok): ((2^29 - 1 - index) << 2) | (4 - kind), index = f * K + k of the
 * first failing (bin, class) (of the problem for pbb_bingham_parameters); at one index the
 * smallest kind is kept (the cause, not the non-finite values a failed class leaves for the
 * later iterations); kind
 *   1: a scatter eigenvalue is negative or numerically zero, i.e. not above 1e-12 times
 *      the largest (the reference asserts >= 0, complex_bingham.py:584; LAPACK and the
 *      Jacobi solver round the zero eigenvalues of a rank-deficient scatter differently)
 *      -> AssertionError;
 *   2: infeasible start of the solve (a zero or negative scatter eigenvalue makes
 *      x0 = -inf or > -1e-8, :378-408) -> ValueError;
 *   3: non-finite scatter, parameters or normaliser -> AssertionError. */
size_t pbb_cbmm_workspace_bytes(int F, int T, int D, int K);

/* CBMMTrainer.fit / _fit / _m_step (cbmm.py:79-237, complex_bingham.py:567-594).
 * init_aff (F, K, T) is required (cbmm.py:120-126 draws it on the host); saliency (F, T)
 * or null (ones, cbmm.py:128-129); weight_mode PBB_WEIGHT_TIME or PBB_WEIGHT_CONST;
 * affiliation_eps clips the posteriors of iterations 2.. to [eps, 1 - eps] (cbmm.py:189).
 * All iterations are enqueued on `stream` without host synchronisation. */
int pbb_cbmm_fit(const void* y, int dtype, int F, int T, int D, int K,
                 const double* init_aff, const double* saliency, int iterations,
                 int weight_mode, double affiliation_eps, double eigenvalue_eps,
                 double max_concentration, void* eigenvectors, double* eigenvalues,
                 double* weight, void* workspace, size_t workspace_bytes,
                 int* status, void* stream);

/* CBMM.predict (cbmm.py:26-55): normalises y, affiliation (F, K, T) out.  weight as for
 * pbb_cwmm_predict (every PBB_WEIGHT_* layout but PBB_WEIGHT_FRAME). */
int pbb_cbmm_predict(const void* y, int dtype, int F, int T, int D, int K,
                     const void* eigenvectors, const double* eigenvalues,
                     const double* weight, int weight_mode, double affiliation_eps,
                     double* affiliation, void* workspace, size_t workspace_bytes,
                     int* status, void* stream);

/* ComplexBinghamTrainer.find_eigenvalues_v3 (complex_bingham.py:304-425), batched:
 * scatter_eigenvalues (n, D) in any order -> eigenvalues (n, D) in the same order.
 * eps: the trainer's eignevalue_eps; max_concentration may be +inf. */
int pbb_bingham_parameters(const double* scatter_eigenvalues, int n, int D, double eps,
                           double max_concentration, double* eigenvalues, int* status,
                           void* stream);

/* ComplexBingham.log_norm (complex_bingham.py:80-164): log c of eigenvalues (n, D);
 * eps > 0 applies the gap rule with that eps first, eps <= 0 does not
 * (remove_duplicate_eigenvalues=False; repeated eigenvalues need no special case here). */
int pbb_bingham_log_norm(const double* eigenvalues, int n, int D, double eps,
                         double* log_norm, void* stream);

/* ComplexBingham.log_pdf (complex_bingham.py:59-78): log_pdf (M, T) = Re(y^H B y) - log_norm,
 * B = V diag(lambda) V^H, for y (M, T, D) as given (not normalised), eigenvectors V (M, D, D)
 * complex128, eigenvalues lambda (M, D), log_norm (M). */
int pbb_bingham_log_pdf(const void* y, int dtype, int M, int T, int D, const void* eigenvectors,
                        const double* eigenvalues, const double* log_norm, double* log_pdf,
                        void* stream);

/* ------------------------------------------------------------------------
 * Batched Hermitian eigendecomposition, ascending eigenvalues
 * (np.linalg.eigh as used in complex_angular_central_gaussian.py:95 and
 * pb_bss/utils.py:154).  a: (n, D, D) complex128 (only read), w: (n, D),
 * v: (n, D, D) complex128, columns are eigenvectors.  0 < D <= 64.  Exact
 * under power-of-two scaling: w(2^k a) = 2^k w(a), v(2^k a) = v(a) for even k.
 * status = 1 + index of the first matrix with non-finite input. */
int pbb_heig_batched(const void* a, int n, int D, double* w, void* v,
                     int* status, void* stream);

/* ------------------------------------------------------------------------
 * Beamforming side (pb_bss/extraction/beamformer.py).  All small matrices and
 * vectors are complex128; the observation may be complex64 or complex128.
 */

/* get_power_spectral_density_matrix (beamformer.py:59-160) for observation
 * (F, D, T) and mask (F, K, T) float64 (or NULL: plain average over time,
 * K must be 1).  normalize: divide by max(sum_t mask, 1e-10) (:127-131).
 * psd: (F, K, D, D).  D < 35, K < 20, any F. */
size_t pbb_psd_workspace_bytes(int F, int T, int D, int K);
int pbb_power_spectral_density(const void* observation, int dtype, int F,
                               int D, int T, const double* mask, int K,
                               int normalize, void* psd, void* workspace,
                               size_t workspace_bytes, void* stream);

/* get_gev_vector (beamformer.py:292-411): eigenvector of the largest
 * generalised eigenvalue of (target, noise), normalised like LAPACK zhegvd
 * ITYPE=1 (w^H noise w = 1).  Replaces _c_get_gev_vector
 * (cythonized/get_gev_vector.pyx:42-150); unlike it, matrices are row-major
 * (n, D, D).  status = 1 + index of the first pair whose noise matrix is not
 * positive definite (the Cython code raises ValueError there, :130-147).
 * 0 < D <= 64.  Target times 2^k and noise times 2^j (j even) give exactly
 * 2^(-j/2) w. */
int pbb_gev_batched(const void* target_psd, const void* noise_psd, int n,
                    int D, void* w, int* status, void* stream);

/* np.linalg.solve for a batch: a (n, D, D), b (n, D, R) -> x (n, D, R), partial
 * pivoting.  hermitize != 0 solves with (a + a^H) / 2.  An exactly singular
 * matrix gets the minimum-norm (lstsq) solution for D <= 40 (the reference's
 * fallback, math/solve.py:95-114); status flags one for D > 40.  0 < D, R <= 64.
 * x(2^k a, b) = 2^-k x(a, b) exactly for even k.  Non-finite a gives NaN. */
int pbb_solve_batched(const void* a, const void* b, int n, int D, int R,
                      int hermitize, void* x, int* status, void* stream);

/* get_mvdr_vector (beamformer.py:230-260): w = N^-1 a / (a^H N^-1 a) with the
 * noise PSD hermitised first.  atf (n, D), noise_psd (n, D, D), w (n, D);
 * scratch: n * D complex128. */
int pbb_mvdr(const void* atf, const void* noise_psd, int n, int D, void* w,
             void* scratch, int* status, void* stream);

/* Pieces of get_mvdr_vector_souden (beamformer.py:601-698): phi = solve(noise,
 * target) -> mat = phi / max(trace(phi).real, eps) and, for every candidate
 * reference channel R, the per-bin numerator / denominator of the SNR
 * (num, den: (n, D) complex128) and their sums over the n bins (num_sum, den_sum:
 * (D) complex128) that get_optimal_reference_channel divides (beamformer.py:616-624). */
int pbb_souden(const void* phi, const void* target_psd, const void* noise_psd,
               int n, int D, double eps, void* mat, void* num, void* den,
               void* num_sum, void* den_sum, void* stream);

/* blind_analytic_normalization (beamformer.py:459-488). */
int pbb_blind_analytic_normalization(const void* vector, const void* noise_psd,
                                     int n, int D, void* out, void* stream);

/* Rank-1 PSD approximation a a^H * trace(cov) / trace(a a^H)
 * (get_pca_rank_one_estimate / get_gev_rank_one_estimate, beamformer_wrapper.py:11-69). */
int pbb_rank_one_estimate(const void* vector, const void* covariance, int n,
                          int D, void* out, void* stream);

/* out = matrix @ vector per batch entry (the scaled GEV ATF Phi_nn w, beamformer_wrapper.py:27-46). */
int pbb_matvec_batched(const void* matrix, const void* vector, int n, int D,
                       void* out, void* stream);

/* apply_beamforming_vector (beamformer.py:572-583): out[f][t] = sum_d conj(w[f][d]) mix[f][d][t]. */
int pbb_apply_beamforming_vector(const void* vector, const void* mix, int dtype,
                                 int F, int D, int T, void* out, void* stream);

/* The same for B beamformers per bin that share ONE mix (the K sources of a separation on one STFT; the reference
 * broadcasts the mix in its einsum): vector (B, F, D), mix (F, D, T), out (B, F, T).  B <= 65535, any F. */
int pbb_apply_beamforming_vector_shared(const void* vector, const void* mix, int dtype,
                                        int B, int F, int D, int T, void* out, void* stream);

/* Differentiates pbb_apply_beamforming_vector: grad_vector[f][a] = sum_t mix[f][a][t] conj(g[f][t]) (fixed order over
 * t), grad_mix[f][a][t] = vector[f][a] g[f][t].  grad_out g (F, T); grad_vector (F, D) and grad_mix (F, D, T)
 * complex128, either may be NULL. */
int pbb_apply_beamforming_vector_backward(const void* vector, const void* mix, int dtype, int F, int D,
                                          int T, const void* grad_out, void* grad_vector, void* grad_mix,
                                          void* stream);

/* Differentiates pbb_apply_beamforming_vector_shared: grad_vector (B, F, D) as above; grad_mix (F, D, T) =
 * sum_b vector[b][f][a] g[b][f][t] summed in increasing b, without materialising the broadcast mix. */
int pbb_apply_beamforming_vector_shared_backward(const void* vector, const void* mix, int dtype, int B,
                                                 int F, int D, int T, const void* grad_out,
                                                 void* grad_vector, void* grad_mix, void* stream);

/* Plain np.linalg.solve without the lstsq fallback (get_mvdr_vector_merl,
 * beamformer.py:277): a (n, D, D), b (n, D, R) -> x (n, D, R).  status must not be
 * NULL; it is set to 1 + the index of an exactly singular matrix (a zero pivot,
 * where NumPy raises LinAlgError), whose x is then undefined. */
int pbb_solve_batched_strict(const void* a, const void* b, int n, int D, int R,
                             void* x, int* status, void* stream);

/* ---- Backward passes of the mask-based beamforming chain (torch.autograd in pb_bss_b200).  For a real loss L every
 * gradient follows PyTorch's convention grad z = dL/dRe z + i dL/dIm z.  fp64, fixed-order sums and no atomics, so
 * repeated calls are bitwise identical; each call only enqueues work on `stream` (no status word, no synchronisation).
 * Gradients are written as complex128 / float64; shapes and limits are those of the forward. */

/* Differentiates pbb_power_spectral_density.  With w_kt = mask_kt / max(S_k, 1e-10), S_k = sum_t mask_kt (normalize),
 * mask_kt (normalize = 0) or 1 / T (mask NULL, K = 1), and G_k = grad_psd[f][k]:
 *   grad_observation[f][:, t] = sum_k w_kt (G_k + G_k^H) y_t,
 *   grad_mask[f][k][t] = (Re(y_t^H G_k y_t) - Re<G_k, psd_k>) / S_k while S_k > 1e-10, else Re(y_t^H G_k y_t) / 1e-10,
 *                        and Re(y_t^H G_k y_t) without normalize (<A, B> = sum conj(A_ij) B_ij).
 * psd is the forward's output (F, K, D, D); grad_psd the same shape; grad_observation (F, D, T) complex128 and
 * grad_mask (F, K, T) float64, either may be NULL.  One pass reads the observation once for all K sources. */
int pbb_power_spectral_density_backward(const void* observation, int dtype, int F, int D, int T,
                                        const double* mask, int K, int normalize, const void* psd,
                                        const void* grad_psd, void* grad_observation, double* grad_mask,
                                        void* stream);

/* Differentiates w = mat[:, ref_channel] of pbb_souden, mat = phi / max(lambda, eps), lambda = Re tr phi,
 * phi = N^-1 X (phi: the forward's pbb_solve_batched output, noise_psd: N, grad_w (n, D)); ref_channel is a constant.
 *   grad phi = g e_r^T / lambda - (Re(g^H phi[:, r]) / lambda^2) I (lambda > eps), g e_r^T / eps otherwise;
 *   grad_target_psd = N^-H grad phi (the elimination of pbb_solve_batched on N^H, N is not assumed Hermitian);
 *   grad_noise_psd = -grad_target_psd phi^H.
 * A bin whose N^H meets an exactly zero pivot (a singular N: the forward's minimum-norm branch, which has no such
 * derivative) or holds non-finite values gets NaN gradients; other bins are unaffected.  0 < D <= 64. */
int pbb_souden_backward(const void* phi, const void* noise_psd, const void* grad_w, int n, int D,
                        int ref_channel, double eps, void* grad_target_psd, void* grad_noise_psd,
                        void* stream);

/* Differentiates the top eigenpair (lambda, w) of pbb_gev_batched (b = the noise PSD) and of pbb_heig_batched's last
 * column (b NULL: B = I, the PCA vector and its eigenvalue).  A and B are the Hermitian parts of a and b, as the
 * forwards read them; w (n, D) is the forward's output, w^H B w = 1.
 *
 * An eigenvector is defined up to a per-bin phase, which the forward's Jacobi solver picks by its rotation sequence.
 * The derivative holds that phase fixed to first order, Im(w^H B dw) = 0 (torch.linalg.eigh's backward assumes the
 * same).  With g = grad_w and g_lambda = grad_lambda (NULL: 0), u = sum_{j != top} w_j (w_j^H g) / (lambda - lambda_j):
 *   grad_a = (G_A + G_A^H) / 2,  G_A = u w^H + g_lambda w w^H,
 *   grad_b = (G_B + G_B^H) / 2,  G_B = -lambda u w^H - (Re(w^H g) / 2 + lambda g_lambda) w w^H   (b != NULL).
 * The projector sum_{j != top} w_j w_j^H / (lambda - lambda_j) does not depend on the phase, so it is recomputed with
 * the forward's own device code (the Cholesky and L^-1 A L^-H reduction of pbb_gev_batched, or the hermitisation of
 * pbb_heig_batched, then the same Jacobi solver) rather than solved for with a bordered system; u w^H is formed with
 * the saved w, whose phase a recomputed top vector must not replace.  For a loss that does not change under
 * w -> e^{i theta} w per bin (w w^H, BAN's output power, the rank-1 estimates) this is the exact gradient; for one that
 * does, it is the gradient with each bin's phase held fixed.
 * A bin whose recomputed top eigenvalue is exactly tied with another, whose B is not positive definite, or which holds
 * non-finite values gets NaN gradients; other bins are unaffected.  grad_a, grad_b (n, D, D); 0 < D <= 64. */
int pbb_eigenvector_backward(const void* a, const void* b, const void* w, const void* grad_w,
                             const double* grad_lambda, int n, int D, void* grad_a, void* grad_b,
                             void* stream);

/* Differentiates pbb_mvdr, w = x / s, x = N_h^-1 a, s = a^H x, N_h = (N + N^H) / 2.  x (n, D) is the forward's scratch
 * (N_h^-1 a), w its output.  With t = w^H g:
 *   q = (g - t a) / conj(s),  p = N_h^-1 q,  grad_atf = p - conj(t) w,  grad_noise_psd = -(p x^H + x p^H) / 2.
 * The solve is pbb_solve_batched's elimination on N_h with a zero pivot giving NaN: a singular N (the forward's
 * minimum-norm branch, which has no such derivative) or non-finite N gives NaN gradients in that bin only.
 * grad_atf (n, D), grad_noise_psd (n, D, D); scratch: n * D complex128.  0 < D <= 64. */
int pbb_mvdr_backward(const void* atf, const void* noise_psd, const void* x, const void* w, const void* grad_w,
                      int n, int D, void* grad_atf, void* grad_noise_psd, void* scratch, void* stream);

/* Differentiates pbb_blind_analytic_normalization, out = c w, c = sqrt|nu| / |delta|, nu = w^H N N w,
 * delta = w^H N w, N read as given (not hermitised).  With r = N w, l = N^H w, rho = Re(w^H g),
 * alpha = rho c conj(nu) / (2 |nu|^2), beta = -rho c conj(delta) / |delta|^2:
 *   grad_vector = c g + alpha N r + conj(alpha) N^H l + beta r + conj(beta) l,
 *   grad_noise_psd = conj(alpha) (w r^H + l w^H) + conj(beta) w w^H.
 * delta = 0, where the forward's c is the constant 0: zero gradients.  nu = 0 with delta != 0 (sqrt|nu| has an
 * infinite derivative there): NaN.  grad_vector (n, D), grad_noise_psd (n, D, D); 0 < D <= 1024. */
int pbb_blind_analytic_normalization_backward(const void* vector, const void* noise_psd, const void* grad_out,
                                              int n, int D, void* grad_vector, void* grad_noise_psd,
                                              void* stream);

/* Differentiates pbb_rank_one_estimate, out = a a^H t / nu, t = sum_d cov_dd (the complex trace), nu = |a|^2.  With
 * G = grad_out and q = a^H G a:
 *   grad_vector = (conj(t) G a + t G^H a) / nu - 2 Re(t conj(q)) / nu^2 a,   grad_covariance = (q / nu) I.
 * |a| = 0 gives NaN in that bin.  grad_vector (n, D), grad_covariance (n, D, D); 0 < D <= 64. */
int pbb_rank_one_estimate_backward(const void* vector, const void* covariance, const void* grad_out, int n,
                                   int D, void* grad_vector, void* grad_covariance, void* stream);

/* Differentiates pbb_matvec_batched, y = M x:  grad_matrix = g x^H,  grad_vector = M^H g.  0 < D <= 64. */
int pbb_matvec_batched_backward(const void* matrix, const void* vector, const void* grad_out, int n, int D,
                                void* grad_matrix, void* grad_vector, void* stream);

/* get_lcmv_vector (beamformer.py:414-456): atf (K, F, D), response (K)
 * complex128 on the device, noise_psd (F, D, D) -> w (F, D).  X = solve(noise, H)
 * with the K ATFs as right-hand sides, y = solve(H^H X, r), w = X y; both solves
 * with stable_solve semantics (pbb_solve_batched).  Like the reference (:444), r is
 * rounded to complex64 first, so a response of 1e-3 is met as float32(1e-3).
 * When any bin's K x K system is exactly singular, y of every bin is rounded to
 * complex64, as the reference's stable_solve does there (it writes into
 * zeros_like(r), math/solve.py:107-113).  scratch: F (2 D K + K K + 2 K) + 1
 * complex128.  status = 1 + a bin whose system is singular with D > 40 or K > 40
 * (no minimum-norm fallback there). */
int pbb_lcmv(const void* atf, const void* response, const void* noise_psd, int K,
             int F, int D, void* w, void* scratch, int* status, void* stream);

/* The filter of get_wmwf_vector (beamformer.py:701-742): phi = stable_solve(noise,
 * target), lambda = trace(phi) (complex, not clamped); filter = phi / (mu + lambda)
 * or, frequency_dependent != 0, phi / sqrt(target[0][0] lambda) (principal root).
 * target_psd, noise_psd, filter (n, D, D); scratch: n D D complex128.  status as
 * pbb_solve_batched.  The caller selects a column or calls pbb_weighted_channel_sum. */
int pbb_wmwf(const void* target_psd, const void* noise_psd, int n, int D,
             int frequency_dependent, double distortion_weight, void* filter,
             void* scratch, int* status, void* stream);

/* out[m][r] = sum_c filter[m][r][c] * weight[m][r][c]: the channel_selection_vector
 * sum of get_wmwf_vector (beamformer.py:743-745).  filter, weight (n, D, D). */
int pbb_weighted_channel_sum(const void* filter, const void* weight, int n, int D,
                             void* out, void* stream);

/* The SNR terms of get_optimal_reference_channel (beamformer.py:601-624) for
 * w_mat (n, D, D): num[m][R] = w_R^H target w_R, den[m][R] = w_R^H noise w_R with
 * w_R = w_mat[m][:, R] (n, D), and their sums over the n bins in bin order
 * (num_sum, den_sum: D complex128).  The same quadratic forms as pbb_souden. */
int pbb_reference_channel_snr(const void* w_mat, const void* target_psd,
                              const void* noise_psd, int n, int D, void* num,
                              void* den, void* num_sum, void* den_sum, void* stream);

/* get_mvdr_vector_merl (beamformer.py:263-289): G = solve(noise, target) with
 * np.linalg.solve (no fallback: status = 1 + a singular bin, the reference raises
 * LinAlgError), w = (G / trace G)[:, 0].  The reference's SNR is summed over the
 * channel axis as well (np.sum of an einsum that keeps only 'c'), so its argmax is
 * always 0 and w is column 0 -- the WMWF filter with mu = 0; no SNR is computed.
 * target_psd, noise_psd (n, D, D), w (n, D), scratch n D D complex128. */
int pbb_mvdr_merl(const void* target_psd, const void* noise_psd, int n, int D,
                  void* w, void* scratch, int* status, void* stream);

/* condition_covariance (beamformer.py:563-569): (x + gamma trace(x) / D I) /
 * (1 + gamma) with the complex trace; x, out (n, D, D). */
int pbb_condition_covariance(const void* x, int n, int D, double gamma, void* out,
                             void* stream);

/* distortionless_normalization (beamformer.py:491-499): out = N w w^H a / (w^H N w);
 * vector, atf, out (n, D), noise_psd (n, D, D). */
int pbb_distortionless_normalization(const void* vector, const void* atf,
                                     const void* noise_psd, int n, int D,
                                     void* out, void* stream);

/* mvdr_snr_postfilter (beamformer.py:502-509): out[m] = (w^H T w) / (w^H N w);
 * vector (n, D), target_psd, noise_psd (n, D, D), out (n). */
int pbb_mvdr_snr_postfilter(const void* vector, const void* target_psd,
                            const void* noise_psd, int n, int D, void* out,
                            void* stream);

/* zero_degree_normalization (beamformer.py:512-514): out = w exp(-i angle(w[ref]))
 * per row; vector, out (n, D). */
int pbb_zero_degree_normalization(const void* vector, int n, int D,
                                  int reference_channel, void* out, void* stream);

/* phase_correction (beamformer.py:517-560): bin f >= 1 is multiplied by the
 * cumulative product of exp(i angle(sum_d conj(w_f[d]) w_{f-1}[d])) along the
 * reference's AXIS 0 OF THE WHOLE ARRAY.  scan_bins = 1 (A = M = 1): a 2-D (F, D)
 * input, axis 0 is the bin axis and the product runs over the bins.  scan_bins = 0:
 * an (A, M, F, D) input (A = axis 0, M = the dims between), and the product runs
 * over A for every (m, f) on its own -- for a (K, F, D) input over the K vectors,
 * not over the bins.  This is the reference's behaviour and is kept.  Row f = 0 is
 * copied; out must not alias vector. */
int pbb_phase_correction(const void* vector, int A, int M, int F, int D,
                         int scan_bins, void* out, void* stream);

/* apply_online_beamforming_vector (beamformer.py:586-598): time-varying filters,
 * out[b][f][t] = sum_d conj(v[t][f][d]) mix[b][f][d][t]; vector complex128,
 * mix complex64 or complex128 (dtype), out (B, F, T) complex128.  Strides in
 * elements: the vector's d stride is 1, frame / bin strides as given (bin stride 0
 * broadcasts one vector bin); the mix's d / t strides are T / 1, batch / bin
 * strides as given (0 broadcasts).  The vector is read once for all B. */
int pbb_apply_online_beamforming_vector(const void* vector, const void* mix,
                                        int dtype, int B, int F, int D, int T,
                                        long long vector_frame_stride,
                                        long long vector_bin_stride,
                                        long long mix_batch_stride,
                                        long long mix_bin_stride, void* out,
                                        void* stream);

/* ------------------------------------------------------------------------
 * Oracle masks (pb_bss/extraction/mask_module.py) and array geometry
 * (pb_bss/extraction/beamform_utils.py), csrc/api_mask.cu.
 *
 * The masks read the signal in its own layout: a pbb_mask_layout describes an
 * index space (row-major over `shape`) and, for every dim, the stride of the
 * input (in elements of the input dtype, complex elements counted once) and of
 * the output.  Inputs may be complex or real (dtype PBB_C64 / PBB_C128 /
 * PBB_F32 / PBB_F64); the arithmetic is fp64, and |s|^2 is re*re + im*im
 * rounded like NumPy (no FMA).  Real-valued masks are stored as float for the
 * 32-bit dtypes and double otherwise.
 */
#define PBB_F32 2
#define PBB_F64 3
#define PBB_MASK_MAX_DIMS 8

typedef struct pbb_mask_layout {
  int nd; /* 0 <= nd <= PBB_MASK_MAX_DIMS; nd = 0 is a single index */
  int reserved;
  long long shape[PBB_MASK_MAX_DIMS];
  long long in_stride[PBB_MASK_MAX_DIMS];
  long long out_stride[PBB_MASK_MAX_DIMS];
} pbb_mask_layout;

/* Source-reduction masks; kind: */
enum {
  PBB_MASK_IDEAL_BINARY = 0,    /* ideal_binary_mask (mask_module.py:90-136): 1 at the first argmax */
  PBB_MASK_WIENER_LIKE = 1,     /* wiener_like_mask (:139-179): p / (sum_k p + eps) */
  PBB_MASK_IDEAL_RATIO = 2,     /* ideal_ratio_mask (:182-232): |s| / (sum_k |s| + eps) */
  PBB_MASK_IDEAL_AMPLITUDE = 3, /* ideal_amplitude_mask (:235-287): |s| / (|sum_k s| + eps) */
  PBB_MASK_PHASE_SENSITIVE = 4, /* phase_sensitive_mask (:290-322): |s| / (|o| + eps) cos(angle s - angle o) */
  PBB_MASK_IDEAL_COMPLEX = 5    /* ideal_complex_mask (:325-347): s / o, NumPy's complex division, no eps */
};
/* For every index r of `rest` (the dims other than the source and sensor axes)
 * and source k: p = sum over the D sensors (channel order; D = 1 without
 * sensor pooling, which only kinds 0 and 1 allow) of |s|^2 at
 * signal + rest.in(r) + k source_stride + d sensor_stride, o = sum_k s.  The
 * mask goes to out + rest.out(r) + k out_source_stride; kind 5 stores the
 * input's element type, the others a real of its precision. */
int pbb_source_mask(const void* signal, int dtype, int kind, int K, int D,
                    long long source_stride, long long sensor_stride,
                    long long out_source_stride, const pbb_mask_layout* rest,
                    double eps, void* out, void* stream);

/* Rows of at most this many elements are selected by one warp in shared
 * memory, several rows per CTA (read in tiles of consecutive rows, so that a
 * row stride of 1 -- the frequency axis of an (F, T) STFT -- coalesces);
 * longer rows are spread over several CTAs per row with histograms in global
 * memory and a pass kernel per digit (scratch: pbb_row_select_scratch_bytes). */
#define PBB_ROW_SELECT_SHORT_MAX 4096
size_t pbb_row_select_scratch_bytes(long long rows, long long n);

/* lorenz_mask (mask_module.py:350-417): each row (index space `rows`, elements
 * `elems`, n = product of elems.shape) holds p = sum over the D sensors of
 * |s|^2 (sensor_stride between them).  The threshold is the smallest of the
 * descending-sorted values whose Lorenz value cumsum / sum is < lorenz_fraction,
 * found by a radix select over the bit patterns of the non-negative doubles
 * (8 digits of 8 bits) that carries per-bucket counts, sums and maxima; the
 * mask stores mask_high where p > threshold, else mask_low.  A row where no
 * value qualifies (np.min of an empty array) sets *status = 1 + its index
 * (the first such row).  Bucket sums are accumulated with atomics, so a
 * Lorenz value within a few ulp of lorenz_fraction may round either way. */
int pbb_lorenz_mask(const void* signal, int dtype, int D, long long sensor_stride,
                    const pbb_mask_layout* rows, const pbb_mask_layout* elems,
                    double lorenz_fraction, double mask_low, double mask_high,
                    void* out, void* scratch, size_t scratch_bytes, int* status,
                    void* stream);

/* quantile_mask (mask_module.py:420-493) for one quantile: x = |s| of every row
 * (rounded to float for the 32-bit dtypes, as np.abs does), the order
 * statistics k_lower and k_upper (0-based, ascending) selected exactly, and
 * np.percentile's linear interpolation (numpy _lerp) evaluated in the input
 * precision: x_lo + (x_hi - x_lo) gamma, or x_hi - (x_hi - x_lo) one_minus_gamma
 * when gamma >= 0.5.  The caller computes k_lower, k_upper, gamma and
 * one_minus_gamma as NumPy does.  mask_high where x > threshold (below = 0) or
 * x < threshold (below = 1), else mask_low. */
int pbb_quantile_mask(const void* signal, int dtype, const pbb_mask_layout* rows,
                      const pbb_mask_layout* elems, long long k_lower,
                      long long k_upper, double gamma, double one_minus_gamma,
                      int below, double mask_low, double mask_high, void* out,
                      void* scratch, size_t scratch_bytes, void* stream);

/* biased_binary_mask (mask_module.py:496-550) with components = 2: for every
 * index r of `rest` (signal without the component axis), p0 / p1 = |s|^2 of
 * component 0 / 1 (component_stride apart) and j = r mod L (the last axis):
 * speech = p0 / speech_div[j] > p1 and > 0.005, noise = p0 / noise_div[j] < p1
 * or < 0.005; force[j] != 0 sets speech = 0, noise = 1.  out (uint8 / bool) gets
 * speech at rest.out(r) and noise at rest.out(r) + out_component_stride.
 * speech_div, noise_div (L doubles) and force (L bytes) are device arrays. */
int pbb_biased_binary_mask(const void* signal, int dtype, long long component_stride,
                           long long out_component_stride, const pbb_mask_layout* rest,
                           int L, const double* speech_div, const double* noise_div,
                           const unsigned char* force, void* out, void* stream);

/* get_steering_vector (beamform_utils.py:36-63): out[a][m][f] (A, M, F)
 * complex128 = exp(-2j pi freq[f] tdoa[a][m]) with NumPy's operation order;
 * normalize != 0 divides by the 2-norm over m (the reference's axis -2). */
int pbb_steering_vector(const double* tdoa, int A, int M, const double* freq, int F,
                        int normalize, void* out, void* stream);

/* get_diffuse_noise_psd (beamform_utils.py:66-97): out (F, D, D) float64 =
 * np.sinc(2 freq[f] distances[d][e] / sound_velocity), sinc(0) = 1. */
int pbb_diffuse_noise_coherence(const double* distances, int D, const double* freq,
                                int F, double sound_velocity, double* out,
                                void* stream);

/* get_nearfield_time_of_flight (beamform_utils.py:100-116): out[s][m] (S, M) =
 * |source[:, s] - sensor[:, m]| / sound_velocity; source (3, S), sensor (3, M).
 * get_farfield_time_difference_of_arrival (:119-159): out[m][k] (M, K) =
 * (sensor[:, m] - sensor[:, reference_channel]) . u_k / sound_velocity with u_k
 * = -(rotate_y(elevation) rotate_z(azimuth))[:, 0]; angles (2, K).  One kernel
 * serves both (mode 0 = near field, 1 = far field; `points` is source or angles). */
int pbb_array_geometry(int mode, const double* points, int S, const double* sensor,
                       int M, int reference_channel, double sound_velocity,
                       double* out, void* stream);

/* ------------------------------------------------------------------------
 * STFT / iSTFT (nara_wpe.utils.stft / istft, as restated in oracle/transform_oracle.py) and the Griffin-Lim / MISI
 * step of pb_bss/transform/griffin_lim_module.py.  size is a power of two in [64, 4096], 1 <= shift <=
 * window_length <= size.  All arithmetic is fp64; twiddle is the host-built table (cos, sin)(2 pi k / size), k < size,
 * as size double pairs.  Spectra are (rows, frames, size/2 + 1) complex128, frame-major.
 */

/* Host only: the frames per CTA (fpc) of the forward and inverse kernels for rows x frames frames of `size` points on
 * a GPU with `sms` SMs.  fpc starts at 4096 / size (two 32 KB ping-pong buffers) and is halved while
 * rows * ceil(frames / fpc) < 2 sms.  pbb_stft, pbb_istft and pbb_griffin_lim_stft launch with this value for the
 * current device.  A frame's arithmetic does not depend on fpc. */
int pbb_stft_frames_per_cta(int size, long long rows, int frames, int sms);

/* nara_wpe stft: frame t of row r holds x[r][t shift - offset + j] * window[j] for j < window_length (zero outside
 * [0, n): offset = window_length - shift with fading, else 0; the end padding of pad=True is the same zero read), then
 * rfft(frame, n=size) -> out[r][t].  x (rows, n) float32 (dtype PBB_F32) or float64 (PBB_F64); window (wl) float64.
 * Replaces the np.pad / segment_axis / einsum / rfft sequence of nara_wpe.utils.stft.  x may be null when n = 0. */
int pbb_stft(const void* x, int dtype, long long rows, long long n, int size, int shift,
             int window_length, int offset, int frames, const double* window,
             const double* twiddle, void* out, void* stream);

/* GriffinLim.step / MISI.step (griffin_lim_module.py:63-66, 112-130), the STFT half: X_dash_dash = stft(x) and, in
 * the same pass, X_dash = |X| exp(i angle(X_dash_dash)) (exp(i angle(0)) = 1).  y == NULL: Griffin-Lim, x = x_hat
 * (K, n).  y != NULL (n float64): MISI, x = x_hat + (y - sum_k x_hat) / K with the sum in row order.  X, X_dash_dash
 * and X_dash are (K, frames, size/2 + 1) complex128.  The iSTFT half is pbb_istft.  With n = 0, x_hat and y may be
 * null (every frame of x is zero, so both forms give X_dash_dash = 0 and X_dash = |X|). */
int pbb_griffin_lim_stft(const double* x_hat, int K, long long n, const double* y,
                         const void* X, int size, int shift, int window_length, int offset,
                         int frames, const double* window, const double* twiddle,
                         void* X_dash_dash, void* X_dash, void* stream);

/* nara_wpe istft: frame_t = irfft(X[r][t], n=size)[:window_length] * synthesis_window (the imaginary parts of the DC
 * and Nyquist bins are ignored), overlap-added into frames * shift + window_length - shift samples in increasing t
 * from 0.0 (the order of np.add.at; no atomics), of which out[r] (n_out float64) receives those from crop on
 * (crop = window_length - shift with fading).  synthesis_window (wl) is nara_wpe's biorthogonal window.  The windowed
 * frames go to workspace (pbb_istft_workspace_bytes).  Replaces the irfft / np.add.at sequence of
 * nara_wpe.utils.istft. */
size_t pbb_istft_workspace_bytes(long long rows, int frames, int window_length);
int pbb_istft(const void* X, long long rows, int frames, int size, int shift, int window_length,
              int crop, long long n_out, const double* synthesis_window, const double* twiddle,
              void* workspace, size_t workspace_bytes, double* out, void* stream);

/* Differentiates pbb_stft wrt x (same arguments; grad_X (rows, frames, size/2 + 1) complex128 is the gradient of out).
 * Per frame dL/dframe_j = size irfft(G^)_j, G^_k = G_k / 2 for 0 < k < size/2 and G_k at k = 0 and size/2, times
 * window[j], then overlap-added in increasing t over the frames covering each sample of [0, n) (fading offset and the
 * pad=False remainder as in the forward; a sample no frame covers gets 0).  grad_x (rows, n) float64.  The frames go
 * to workspace (pbb_stft_backward_workspace_bytes). */
size_t pbb_stft_backward_workspace_bytes(long long rows, int frames, int window_length);
int pbb_stft_backward(const void* grad_X, long long rows, long long n, int size, int shift,
                      int window_length, int offset, int frames, const double* window,
                      const double* twiddle, void* workspace, size_t workspace_bytes, double* grad_x,
                      void* stream);

/* Differentiates pbb_istft wrt X (same arguments; grad_out (rows, n_out) float64 is the gradient of out).  The STFT
 * of the gradient: frame t reads grad_out[t shift + j - crop] (zero outside [0, n_out)) times synthesis_window[j],
 * h = that frame, and grad_X[r][t][k] = (2 / size) rfft(h)_k for 0 < k < size/2, (1 / size) Re rfft(h)_k with a zero
 * imaginary part at k = 0 and size/2.  grad_X (rows, frames, size/2 + 1) complex128. */
int pbb_istft_backward(const double* grad_out, long long rows, int frames, int size, int shift,
                       int window_length, int crop, long long n_out, const double* synthesis_window,
                       const double* twiddle, void* grad_X, void* stream);

/* ------------------------------------------------------------------------
 * Gammatone filterbank (pb_bss/transform/gammatone.py:6-102, Slaney's Apple TR #35), csrc/gammatone.cuh.
 *
 * Filter i is a cascade of four second-order sections with numerators [b0_k, b1_k, 0] and the shared denominator
 * [1, a1, a2], each run from zero state in direct form II transposed (scipy.signal.lfilter).  The cascade is one
 * linear recurrence with 8 states, made parallel over time by a scan over chunks of L samples: the zero-start end
 * state of every (row, filter, chunk), a carry s_{c+1} = M s_c + z_c over the chunks (M = the cascade's zero-input
 * transition over L samples), and a rerun of every chunk from its carried start state that writes the output.  All
 * fp64, no atomics (bitwise reproducible).
 *
 * L is the largest power of two in [PBB_GAMMATONE_CHUNK_MIN, PBB_GAMMATONE_CHUNK_MAX] that still gives at least
 * PBB_GAMMATONE_MIN_CHUNKS (row, filter, chunk) sequences, else PBB_GAMMATONE_CHUNK_MIN; a host-only function of
 * the shape.  Signals of at most L samples are one chunk and skip the scan. */
#define PBB_GAMMATONE_CHUNK_MIN 128
#define PBB_GAMMATONE_CHUNK_MAX 1024
#define PBB_GAMMATONE_MIN_CHUNKS 65536
#define PBB_GAMMATONE_CARRY_GROUP 32 /* chunks per group of the two-level carry: M^32 is the group transition */
int pbb_gammatone_chunk_length(long long rows, int n, long long N);
/* Bytes of the scan's state workspace (0 when N fits one chunk). */
size_t pbb_gammatone_workspace_bytes(long long rows, int n, long long N);
/* x (rows, N) float32 (dtype PBB_F32) or float64 (PBB_F64), contiguous; out (n, rows, N) float64.
 * coef (n, 10) float64: b0_0, b1_0, ..., b0_3, b1_3, a1, a2 per filter.  transition (n, 2, 8, 8) float64, row-major:
 * M and M^PBB_GAMMATONE_CARRY_GROUP on the state vector (u_0, v_0, ..., u_3, v_3) of the four sections, where a
 * section with input w and output y = b0 w + u updates u <- b1 w + v - a1 y, v <- -a2 y.  chunk_length must be
 * pbb_gammatone_chunk_length(rows, n, N): M depends on it. */
int pbb_gammatone(const void* x, int dtype, long long rows, long long N, int n, const double* coef,
                  const double* transition, int chunk_length, void* workspace, size_t workspace_bytes,
                  double* out, void* stream);

/* ------------------------------------------------------------------------
 * SRMR, the speech-to-reverberation modulation energy ratio (pb_bss/evaluation/module_srmr.py:42-186), csrc/srmr.cuh
 * and csrc/fft_large.cuh.  One pass per step of the reference, every row of a batch at once; all sizes derive from
 * N, and the per-row lengths N_r after the VAD stay on the device.  fp64 (the VAD's threshold compare in the input
 * precision), no float atomics: bitwise reproducible, and a row's results do not depend on the rest of the batch. */
#define PBB_SRMR_MAX_SAMPLES 4194304 /* 2^22 */
#define PBB_SRMR_VAD_TILE 4096       /* samples per CTA of the VAD passes */
/* _preprocessing_vad (:158-186) and the normalisation (:58-60).  x (rows, N) float32 (PBB_F32) or float64 (PBB_F64).
 * threshold = max|x|^2 / 1e5 in x's precision; the samples strictly between two above-threshold samples more than
 * `gap` (0.05 sample_rate) apart are removed.  out (rows, N) float64: the kept samples of each row at its start, zero
 * after; nr (rows) long long: N_r.  normalise != 0: out becomes (out - mean) / std (population std) over the first N_r
 * samples; stats (rows, 2) float64 gets mean and std (either way, unused entries when normalise = 0). */
size_t pbb_srmr_vad_workspace_bytes(long long rows, long long N);
int pbb_srmr_vad(const void* x, int dtype, long long rows, long long N, double gap, int normalise, void* workspace,
                 size_t workspace_bytes, double* out, long long* nr, double* stats, void* stream);
/* |scipy.signal.hilbert(y[s, :N_r])| (:65-67) of every sequence s = f rows + r of y (n rows, N) float64, in place
 * (entries past N_r are left as they are).  The imaginary part of the analytic signal is y convolved with the
 * discrete Hilbert kernel of length N_r, one real FFT of M = 2P = nextpow2(2N - 1) points per sequence (at least 2),
 * computed as a four-step complex FFT of P points in global memory.  `group` sequences are transformed at a time,
 * which sets the workspace (pbb_srmr_hilbert_workspace_bytes); the result does not depend on it. */
int pbb_srmr_fft_log2(long long N); /* log2 M */
size_t pbb_srmr_hilbert_workspace_bytes(long long rows, long long N, long long group);
int pbb_srmr_hilbert(double* y, long long rows, long long N, int n, const long long* nr, long long group,
                     void* workspace, size_t workspace_bytes, void* stream);
/* The modulation filterbank and energies (:70-118): means (rows, n, 8) float64 of the Hamming-windowed frame energies
 * of the eight modulation filters over the first N_r samples of every envelope env (n rows, N).  hop = int(sr / 1000)
 * * 64, frames of 4 hop.  coef (8, 3): b0, a1, a2 of b = [b0, 0, -b0], a = [1, a1, a2].  transition (8, 4): the
 * filter's zero-input state transition over hop samples, row-major 2 x 2 on (z0, z1) of lfilter's direct form II
 * transposed.  window (4 hop): scipy.signal.windows.hamming(4 hop, sym=True). */
size_t pbb_srmr_means_workspace_bytes(long long rows, long long N, int n, int hop);
int pbb_srmr_means(const double* env, long long rows, long long N, int n, const long long* nr, int hop,
                   const double* coef, const double* transition, const double* window, void* workspace,
                   size_t workspace_bytes, double* means, void* stream);
/* The ratio (:104-154): out (rows) float64 from means (rows, n, 8), erb (n) = cfs / 9.26449 + 24.7 and cutoff (8). */
int pbb_srmr_ratio(const double* means, long long rows, int n, const double* erb, const double* cutoff, double* out,
                   void* stream);

/* ------------------------------------------------------------------------
 * BSS Eval v3 (Vincent, Gribonval and Fevotte 2006), mir_eval_sources of pb_bss/evaluation/module_mir_eval.py:5-141:
 * mir_eval.separation.bss_eval_sources and its _bss_decomp_mtifilt / _project / _bss_source_crit with 512-tap
 * time-invariant distortion filters, and pb_bss's _bss_eval_sources_and_noise (:94-141) for K + 1 estimates.
 * csrc/bss_eval.cuh.  fp64 throughout, no float atomics: bitwise reproducible, and an item's results do not depend
 * on the rest of the batch or on `group`.
 *
 * x (items, K + E, T) float64: per item the K references, then the E estimates (E = K or K + 1).  For every item
 * the lag correlations r_ab[d] = sum_u a[u] b[u + d] (d < 512) on the fp64 tensor cores, the system G c = D of
 * order N = 512 K (G[(i,t1),(j,t2)] = r_ij[t1 - t2], D[(i,t), e] = r_(i, estimate e)[t]) and the K diagonal blocks
 * are factored ONCE each by LU with partial pivoting (mir_eval solves per (estimate, reference) pair), and the sums
 * of squares of the explicit residual signals P_j x, x - P_j x, P_all x - P_j x, P_all x and x - P_all x over T + 511
 * samples give SDR / SIR / SAR of every (estimate e, reference j) pair with mir_eval's _safe_db (a zero denominator
 * gives +inf, a zero numerator over a positive one -inf).
 * compute_permutation != 0: sdr / sir / sar / selection (items, K) of the first maximiser, in
 * itertools.permutations(range(E), K) order, of the mean SIR (np.mean's summation order; np.argmax: the first NaN
 * wins).  compute_permutation = 0 (needs E = K): the pairs (k, k); selection is not written (may be null).
 * pairs (items, 3, E, K) float64, may be null: SDR, SIR, SAR of every pair.
 * *status (long long; set to 0 by the call) = ((item + 1) << 3) | flags of the first failing item, flags: 1 = an
 * all-zero reference or estimate (mir_eval's validate raises ValueError; the reference's K + 1 path would fall
 * through to lstsq), 2 = a non-finite sample, 4 = an exactly zero LU pivot (mir_eval switches to lstsq there).  A
 * failing item's outputs are NaN.  Items run `group` at a time, which sets the workspace
 * (pbb_bss_eval_workspace_bytes: G alone is group * N * (N + 16) * 8 bytes, 135 MB per item at K = 8). */
#define PBB_BSS_EVAL_FILTER 512
#define PBB_BSS_EVAL_MAX_SOURCES 8        /* K <= 8, N <= 4096 (OutputMetrics asserts K <= 8) */
#define PBB_BSS_EVAL_MAX_SAMPLES 4194304  /* 2^22 */
#define PBB_BSS_EVAL_MAX_GROUP 65535
size_t pbb_bss_eval_workspace_bytes(long long group, int K, int E, long long T);
int pbb_bss_eval(const double* x, long long items, int K, int E, long long T, int compute_permutation,
                 long long group, void* workspace, size_t workspace_bytes, double* sdr, double* sir, double* sar,
                 long long* selection, double* pairs, long long* status, void* stream);

/* ------------------------------------------------------------------------
 * STOI, the short-time objective intelligibility (Taal et al. 2011) of pb_bss/evaluation/module_stoi.py:4-25, i.e.
 * pystoi.stoi(x, y, fs_sig) with extended=False, for every row of a batch at once.  csrc/stoi.cuh.  fp64 throughout,
 * no float atomics: bitwise reproducible, and a row's results do not depend on the rest of the batch or on `group`.
 *
 * x (reference) and y (estimate) are (rows, n), both float32 (PBB_F32) or both float64 (PBB_F64), read in place.
 * Per row:
 *  1. up / down != 1 (10000 / fs in lowest terms): scipy.signal.resample_poly(s, 10000, fs, window=h / h.sum()) of x
 *     and y, L = ceil(n up / down) samples.  taps (up, taps_per_phase) float64: taps[ph][m] = hp[ph + m up] (0 past
 *     the end), where hp is resample_poly's filter: the window times up, preceded by its n_pre_pad zeros; pre_remove
 *     is its n_pre_remove.  Output j is sum_m taps[ph][m] x[i0 - m] with t = (j + pre_remove) down, ph = t mod up,
 *     i0 = t / up (x = 0 outside [0, n)).  up = down = 1: L = n, the input is framed as it is; taps may be null.
 *  2. the silent-frame removal (pystoi.utils.remove_silent_frames): F frames f with 128 f < L - 256 (strict),
 *     E_f = 20 log10(||window * x_f|| + eps); frame f is kept where (max E - 40) - E_f < 0 (a NaN max keeps none);
 *     K_r kept frames, M_r = max(K_r - 1, 0) STFT frames of the overlap-added signal.
 *  3. the STFT (pystoi.utils.stft): STFT frame i is kept frames i - 1, i, i + 1 overlap-added, windowed again,
 *     rfft(n=512) with the twiddle table (512 (cos, sin)(2 pi k / 512) pairs, the STFT's convention); band energies
 *     sqrt(sum_{bands[b][0] <= k < bands[b][1]} |X_k|^2) for the 15 one-third octave bands (bands (15, 2) int).
 *     window (256) float64 = np.hanning(258)[1:-1].
 *  4. M_r < 30: out[r] = 1e-5 (pystoi warns and returns 1e-5).  Else the J_r = M_r - 29 segments of 30 frames:
 *     y' = min(y_seg ||x_seg|| / (||y_seg|| + eps), x_seg (1 + 10^(15/20))) (NaN if either is), both mean-removed and
 *     divided by (norm + eps), and out[r] = sum of the inner products over (segment, band) / (J_r 15).
 * out (rows) float64.  frames (rows, 2) long long, may be null: K_r, M_r.  resampled (rows, 2, L) float64, may be
 * null: x and y at 10 kHz (not written at 10 kHz).  energies (rows, 2, 15, M_max = F - 1) float64, may be null: the
 * band energies of x and y (entries from M_r on are not written).  status (2 long long, set by the call): the number
 * of rows with M_r < 30 and the first such row (-1: none).  Rows run `group` at a time, which sets the workspace
 * (pbb_stoi_workspace_bytes; 0 for an invalid shape).  n must be in [1, PBB_STOI_MAX_SAMPLES] and L in
 * (PBB_STOI_FRAME, PBB_STOI_MAX_RESAMPLED]: at most 256 samples at 10 kHz give no frame, where pystoi raises.
 *
 * pbb_estoi: ESTOI, the extended STOI (Jensen and Taal, IEEE/ACM TASLP 24(11), 2016), i.e. pystoi.stoi(x, y, fs_sig,
 * extended=True).  Exactly pbb_stoi's arguments, workspace (pbb_stoi_workspace_bytes), frames / resampled / energies
 * outputs and status words; steps 1-3 and the 1e-5 rule of step 4 are the same bit for bit.  For M_r >= 30, each
 * segment X, Y (15 bands x 30 frames) of the band energies, without clipping or scaling, is normalised per band (minus
 * the mean over the frames, divided by the root of the sum of squares), then per frame (minus the mean over the bands,
 * divided by the root of the sum of squares), and out[r] = the sum of X Y over (segment, band, frame) / (J_r 30).
 * pystoi adds N(0, eps^2) noise before each normalisation; here a row or column whose centred sum of squares is zero
 * up to rounding, at most 2^-92 times its sum of squares before centring, normalises to zeros (digital silence, and
 * the constant columns of a segment of y with one non-zero frame); NaN and inf propagate. */
#define PBB_STOI_FS 10000
#define PBB_STOI_FRAME 256
#define PBB_STOI_NFFT 512
#define PBB_STOI_BANDS 15
#define PBB_STOI_SEGMENT 30
#define PBB_STOI_DYN_RANGE 40
#define PBB_STOI_MAX_SAMPLES 4194304    /* 2^22 */
#define PBB_STOI_MAX_RESAMPLED 8388608  /* 2^23 samples at 10 kHz */
#define PBB_STOI_MAX_GROUP 65535
size_t pbb_stoi_workspace_bytes(long long group, long long n, int up, int down);
int pbb_stoi(const void* x, const void* y, int dtype, long long rows, long long n, int up, int down,
             const double* taps, int taps_per_phase, long long pre_remove, const double* window, const int* bands,
             const double* twiddle, long long group, void* workspace, size_t workspace_bytes, double* out,
             long long* frames, double* resampled, double* energies, long long* status, void* stream);
int pbb_estoi(const void* x, const void* y, int dtype, long long rows, long long n, int up, int down,
              const double* taps, int taps_per_phase, long long pre_remove, const double* window, const int* bands,
              const double* twiddle, long long group, void* workspace, size_t workspace_bytes, double* out,
              long long* frames, double* resampled, double* energies, long long* status, void* stream);

/* pbb_stoi_backward: the gradient of pbb_stoi's (extended = 0) or pbb_estoi's (extended = 1) out with respect to x
 * and y.  x, y, dtype, rows, n, up, down, taps, taps_per_phase, pre_remove, window, bands, twiddle and group are
 * pbb_stoi's; grad_out (rows) float64 is dL/dout; grad_x, grad_y (rows, n) float64 receive dL/dx, dL/dy (every
 * element written; either may be null, and its chain is skipped).  The workspace is
 * pbb_stoi_backward_workspace_bytes(group, n, up, down, extended) (0 for an invalid shape); nothing is kept from the
 * forward: steps 1-3 run again with the forward's kernels, so the keep mask, the kept frames and the band energies
 * are bitwise the forward's.  Only enqueues work (no status word, no host synchronisation); fp64, every sum a gather
 * in a fixed order, no atomics: repeated calls are bitwise identical.
 *
 * The derivative, per row with M_r >= 30 (rows on the 1e-5 path, including a non-finite reference, get zeros):
 *  - the keep mask is a constant (it depends on x only through a threshold): the gradient flows through the kept
 *    frames into x and y; a dropped frame's samples get only what the kept frames over them pass;
 *  - band energies e_b = sqrt(sum_k |X_k|^2): dL/dX_k = (dL/de_b / e_b) X_k, 0 where e_b = 0; the frame gradient is
 *    Re sum_k (dL/dX_k) e^{+2 pi i j k / 512} (j < 256) times the window, then the overlap-add and the first window
 *    are transposed, then the resampler (the polyphase filter's transpose; the identity at 10 kHz);
 *  - STOI, per (segment, band) with g = grad_out / (15 J): c = ||x|| / (||y|| + eps), y' = min(c y, C x) with the
 *    gradient to the operand the forward selected (x on a tie), a = y' - mean, e = x - mean,
 *    d = <a, e> / ((||a|| + eps)(||e|| + eps)): dd/da = e / (Da De) - d a / (Da ||a||), dd/de symmetric, each
 *    mean-removal's transpose, dc/dx = x / (||x|| (||y|| + eps)), dc/dy = -||x|| y / ((||y|| + eps)^2 ||y||); a zero
 *    norm (||x||, ||y||, ||a||, ||e||) has a zero subgradient;
 *  - ESTOI, per segment with g = grad_out / (30 J): z = v / ||v|| after centring, per band then per frame; the
 *    transpose of each step is (I - z z^T) / ||v|| then the centring's; a row or column that the 2^-92 rule
 *    normalises to zeros passes no gradient;
 *  - a non-finite y with a finite x gives NaN gradients (in that row only).  Digital silence in y gives finite
 *    gradients, large where c ~ ||x|| / eps. */
size_t pbb_stoi_backward_workspace_bytes(long long group, long long n, int up, int down, int extended);
int pbb_stoi_backward(const void* x, const void* y, int dtype, long long rows, long long n, int up, int down,
                      const double* taps, int taps_per_phase, long long pre_remove, const double* window,
                      const int* bands, const double* twiddle, long long group, void* workspace,
                      size_t workspace_bytes, int extended, const double* grad_out, double* grad_x, double* grad_y,
                      void* stream);

/* ------------------------------------------------------------------------
 * SI-SDR (pb_bss/evaluation/module_si_sdr.py:4-56) and the invasive SxR (pb_bss/evaluation/sxr_module.py:17-274).
 * csrc/sxr.cuh.  fp64 throughout, no float atomics.  A row of n samples is summed in ceil(n / PBB_SXR_CHUNK) chunks,
 * each in a fixed order inside one CTA, then the chunk partials in a fixed order: the tree depends on n only, so a
 * row's value is bitwise the same in any batch.  Products and differences round as NumPy's do (no FMA); only the order
 * of the length-n sums differs from NumPy's pairwise sum.  Every call only enqueues work on `stream`. */
#define PBB_SXR_CHUNK 8192
#define PBB_SXR_MAX_K 9    /* sxr_module asserts K < 10 */
#define PBB_SXR_MAX_D 29   /* input_sxr asserts D < 30 */
#define PBB_I16 4
#define PBB_I32 5
#define PBB_I64 6
/* get_variance_for_zero_mean_signal (:17-23) over the last axis: out[r] = mean |x[r, :]|^2, float64 (rows).  x (rows, n)
 * contiguous, dtype PBB_F32 / PBB_F64 / PBB_I16 / PBB_I32 / PBB_I64 (x^2 in fp64) or PBB_C64 / PBB_C128 (re re + im im).
 * n = 0 gives NaN (np.mean of nothing) and x may then be null.  Workspace: rows * chunks doubles
 * (pbb_mean_square_workspace_bytes; may be null when that is 0). */
size_t pbb_mean_square_workspace_bytes(long long rows, long long n);
int pbb_mean_square(const void* x, int dtype, long long rows, long long n, void* workspace, size_t workspace_bytes,
                    double* out, void* stream);
/* si_sdr (:38-56) per row: alpha = <r, e> / <r, r> (pass 1), then 10 log10(sum (alpha r)^2 / sum (e - alpha r)^2) from
 * the rounded projection alpha r and residual e - alpha r (pass 2), with the same summation tree for every sum: e = 2^j r
 * gives alpha = 2^j, a zero residual and +inf; a zero reference or estimate gives NaN.  reference / estimation float64,
 * row r at reference + reference_offsets[r] and estimation + estimation_offsets[r] (device int64 element offsets, so a
 * broadcast operand is not materialised), n contiguous samples each.  Workspace: pbb_si_sdr_workspace_bytes. */
size_t pbb_si_sdr_workspace_bytes(long long rows, long long n);
int pbb_si_sdr(const double* reference, const double* estimation, const long long* reference_offsets,
               const long long* estimation_offsets, long long rows, long long n, void* workspace,
               size_t workspace_bytes, double* out, void* stream);
/* Differentiates pbb_si_sdr (same first six arguments, grad_out (rows) float64).  With p = alpha r and q = e - p as
 * pass 2 forms them, P = sum p^2, Q = sum q^2: ds/de = (20 / ln 10)(p / P - q / Q), ds/dr = (20 alpha / ln 10)
 * (1 / P + 1 / Q) q.  A broadcast operand's gradient sums the rows that read it: own row u of the reference
 * (reference_rows of them, n samples each) is the sum over the rows reference_row_index[reference_row_start[u]] ..
 * [reference_row_start[u + 1] - 1] in that order (device int64 tables); the same for the estimation.  grad_reference /
 * grad_estimation (own rows, n) float64, either may be NULL.  inf / NaN rows (zero reference, e = 2^j r, ...) give
 * non-finite gradients.  Workspace: pbb_si_sdr_backward_workspace_bytes. */
size_t pbb_si_sdr_backward_workspace_bytes(long long rows, long long n);
int pbb_si_sdr_backward(const double* reference, const double* estimation, const long long* reference_offsets,
                        const long long* estimation_offsets, long long rows, long long n, const double* grad_out,
                        long long reference_rows, const long long* reference_row_start,
                        const long long* reference_row_index, long long estimation_rows,
                        const long long* estimation_row_start, const long long* estimation_row_index, void* workspace,
                        size_t workspace_bytes, double* grad_reference, double* grad_estimation, void* stream);
/* input_sxr (:94-165) from the powers S (K, D) and N (D), float64 on the device, in the reference's order of
 * operations: I[k, d] = np.sum of S[n != k, d], the channel means (average_channels), S / (I + N), S / I, S / N in dB
 * (IEEE inf / nan for zero powers), then the source mean (average_sources).  sdr / sir / snr have the shape of the
 * result: (K, D), (K), (D) or one value.  np.sum of fewer than 8 values is a left-to-right loop, from 8 on NumPy's
 * 8-accumulator pairwise pattern; np.mean(axis=0) of (K, D > 1) adds the rows in order.  1 <= K <= PBB_SXR_MAX_K,
 * 1 <= D <= PBB_SXR_MAX_D. */
int pbb_input_sxr(const double* S, const double* N, int K, int D, int average_sources, int average_channels,
                  double* sdr, double* sir, double* snr, void* stream);
/* output_sxr (:168-274) from S (K_source, K_target) and N (K_target): the mutual power np.sum(S[k, p[k]]) of every
 * p of itertools.permutations(range(K_target), K_source) (up to 9! = 362880, unranked in parallel), the first maximiser
 * as np.argmax picks it (a NaN wins), then SDR / SIR / SNR (K_source, or their means with average_sources) and
 * selection (K_source) int64.  1 <= K_source <= K_target <= PBB_SXR_MAX_K.  Workspace:
 * pbb_output_sxr_workspace_bytes. */
size_t pbb_output_sxr_workspace_bytes(int K_source, int K_target);
int pbb_output_sxr(const double* S, const double* N, int K_source, int K_target, int average_sources, void* workspace,
                   size_t workspace_bytes, double* sdr, double* sir, double* snr, long long* selection, void* stream);

/* ------------------------------------------------------------------------
 * k-means of BinaryGMMTrainer (pb_bss/distribution/gmm.py:176-230): sklearn.cluster.KMeans(n_clusters=K) with its
 * defaults (k-means++, n_init='auto' = 1, Lloyd, max_iter 300, tol 1e-4), in fp64.
 */
#define PBB_KMEANS_MAX_K 16
#define PBB_KMEANS_MAX_E 64

/* Workspace of pbb_kmeans_fit: (N (E + 7) + O(256 (K E + K + 2 E))) doubles; 0 for a shape outside the limits. */
size_t pbb_kmeans_workspace_bytes(long long N, int E, int K);
/* KMeans.fit on x (N, E) float64 row-major: X_mean and the centred copy, tol = 1e-4 * mean(var(x, axis=0)), the
 * initial centres, then _kmeans_single_lloyd (the labels as the first argmin of |c|^2 - 2 x.c; strict convergence
 * when no label changed, else stop when the summed squared centre shift is <= tol; the final E-step when not strict;
 * empty clusters relocated as _relocate_empty_clusters_dense, with the farthest points taken largest first, ties to
 * the lower index).  Initial centres: init (K, E) device, raw coordinates, when not null; else _kmeans_plusplus with
 * n_local_trials L = 2 + int(log K) from the host's draws: first = the index of the first centre
 * (random_state.choice), uniforms (K - 1, L) device = the unscaled random_state.uniform draws of the K - 1 rounds.
 * Out: centres (K, E) with X_mean added back, labels (N) int32, inertia, n_iter.  *status (device) is zeroed, then
 * bit 0 = x holds a non-finite value (nothing is fitted), bit 1 = fewer distinct labels than K, with their count in
 * bits 8 and up.  Every sum runs in an order that depends on N only, so the results are bitwise repeatable and
 * do not depend on the grid: max_ctas > 0 caps the CTAs of the two cooperative launches (0 = as many as the device
 * holds at once, up to one per chunk of at most 256).  Relocation follows sklearn: no point moves when the largest
 * distance to an old centre is 0.  Needs a device with cooperative launch (every H100 has it).
 * 1 <= K <= min(N, PBB_KMEANS_MAX_K), 1 <= E <= PBB_KMEANS_MAX_E, N < 2^31. */
int pbb_kmeans_fit(const double* x, long long N, int E, int K, long long first, const double* uniforms,
                   const double* init, int max_iter, void* workspace, size_t workspace_bytes, double* centres,
                   int* labels, double* inertia, int* n_iter, int* status, int max_ctas, void* stream);
/* KMeans.predict: labels (N) int32 = the first argmin of |c|^2 - 2 x.c over centres (K, E); one_hot (K, N) float64
 * (labels_to_one_hot(labels, K, axis=-2)).  Either output may be null. */
int pbb_kmeans_predict(const double* x, long long N, int E, int K, const double* centres, int* labels,
                       double* one_hot, void* stream);

/* ------------------------------------------------------------------------
 * Frequency permutation alignment (pb_bss/permutation_alignment.py).
 */

/* DHTVPermutationAlignment.calculate_mapping (:295-355) with its defaults: pbb_dhtv_mapping_ex with similarity 'cos'
 * and the greedy assignment (:525-553).  mask (K, F, T) float64 is only read;
 * plan: nplan triples (iterations, start, end) as produced by
 * alignment_plan (:204-293) -- a small HOST array (checked and sized on the host,
 * then copied into the scratch); features (K, F, T) and centroid
 * (pbb_dhtv_scratch_doubles doubles) are device scratch; mapping (K, F) int64 out.
 * The reference's early exit is reproduced with device-side flags. */
size_t pbb_dhtv_scratch_doubles(int K, int T, const int* plan, int nplan);
int pbb_dhtv_mapping(const double* mask, int K, int F, int T, const int* plan,
                     int nplan, double* features, double* centroid,
                     long long* mapping, void* stream);
/* The same with the reference's options (permutation_alignment.py:133-163): metric 0 = 'multiply' (raw masks, inner
 * product), 1 = 'cos' (the default: features and centroid L2-normalised over time), 2 = 'euclidean' (minus the
 * distance); algorithm 0 = 'greedy', 1 = 'optimal' (brute force over the K! permutations).  The whole plan runs in
 * one launch: a single thread-block cluster that keeps a segment's feature rows in distributed shared memory when the
 * widest segment fits (<= 16 bins per CTA of a 16- or 8-CTA cluster and <= 200 KB; the reference's plans do), else one
 * cooperative launch with grid-wide barriers.  The two add the centroid in different orders, so the integer mapping
 * is the same on both wherever no decision lies within rounding of a tie, and on exact ties (first maximum in
 * row-major order); tests/test_permutation_gpu.py::test_dhtv_every_kernel_matches_the_oracle checks both against the
 * reference.  K * T * 8 bytes must not exceed 200 KB (the centroid lives in shared memory).  Needs a device with
 * cooperative launch (every H100 has it); elsewhere the call fails with a runtime error before any device work. */
int pbb_dhtv_mapping_ex(const double* mask, int K, int F, int T, const int* plan,
                        int nplan, double* features, double* centroid,
                        long long* mapping, int metric, int algorithm, void* stream);

/* apply_mapping (:54-104): out[k, f, :] = mask[mapping[k, f], f, :]. */
int pbb_apply_mapping(const double* mask, const long long* mapping, int K,
                      int F, int T, double* out, void* stream);

/* _ScoreMatrix.multiply / cos / euclidean (:380-420): scores (F, K, K) with
 * scores[f][k_reference][k_mask] over the T frames of bin f.  Source k of a
 * side starts at base + k * source_stride (elements), its bins are T apart, so
 * the shifted views mask[:, 1:] / mask[:, :-1] of GreedyPermutationAlignment
 * (:702) are passed without a copy.  metric: */
enum { PBB_SCORE_MULTIPLY = 0, PBB_SCORE_COS = 1, PBB_SCORE_EUCLIDEAN = 2 };
int pbb_score_matrix(const double* mask, const double* reference,
                     long long mask_source_stride,
                     long long reference_source_stride, int K, int F, int T,
                     int metric, double* scores, void* stream);

/* _mapping_from_score_matrix (:458-590): scores (F, K, K) -> mapping (K, F)
 * int64.  algorithm 0 = 'greedy', 1 = 'optimal' (first best of
 * itertools.permutations).  *status = 1 + bin of a non-finite score matrix
 * (the reference raises ValueError('score matrix is infeasible')). */
enum { PBB_ASSIGN_GREEDY = 0, PBB_ASSIGN_OPTIMAL = 1 };
int pbb_mapping_from_score_matrix(const double* scores, int F, int K,
                                  int algorithm, long long* mapping,
                                  int* status, void* stream);

/* GreedyPermutationAlignment.calculate_mapping (:700-712), last step:
 * pair_mapping (K, F-1) = mapping of every bin to its lower neighbour;
 * mapping (K, F): column 0 identity, column f = pair[mapping[:, f-1], f-1]. */
int pbb_chain_mapping(const long long* pair_mapping, int K, int F,
                      long long* mapping, void* stream);

/* ------------------------------------------------------------------------
 * Single distributions (pb_bss/distribution/complex_angular_central_gaussian.py, complex_watson.py,
 * complex_circular_symmetric_gaussian.py).  Every model and output is fp64 / complex128; the observation may be
 * complex64 or complex128 (`dtype`).  Model broadcasting over leading dims is resolved by the caller: y_stride is
 * the number of elements between the observations of consecutive models, 0 when all models share one y.
 * ------------------------------------------------------------------------ */

/* ComplexAngularCentralGaussian.from_covariance (complex_angular_central_gaussian.py:81-132) for covariance
 * (n, D, D): covariance_norm PBB_NORM_TRACE divides by max(real trace, tiny) first (into a copy: the input is not
 * changed); the Hermitian part is diagonalised (pbb_heig_batched's Jacobi solver); PBB_NORM_EIGENVALUE scales the
 * eigenvalues by 1 / max(lambda_max, tiny) and floors them at eigenvalue_floor, the other norms floor them at
 * lambda_max * eigenvalue_floor.  eigenvectors (n, D, D) columns, eigenvalues (n, D) ascending.  0 < D <= 64.
 * *status (reset by the call) = 1 + the first matrix with non-finite input or eigenvalues (the reference asserts
 * np.isfinite, :127). */
int pbb_cacg_from_covariance(const void* covariance, int n, int D, int covariance_norm, double eigenvalue_floor,
                             void* eigenvectors, double* eigenvalues, int* status, void* stream);

/* ComplexAngularCentralGaussian._log_pdf (:167-203) from the quadratic forms of pbb_cacgmm_predict: quadratic_out
 * (F, K, T), a buffer of its own, receives max(|q|, q_floor) of quadratic (F, K, T) -- q_floor =
 * np.finfo(y.dtype).tiny -- and log_pdf (F, K, T) = -D log q - sum_d log eigenvalues (F, K, D).  F * K <= 65535.
 * pbb_cacg_log_pdf is this with q_floor = DBL_MIN and no quadratic_out. */
int pbb_cacg_log_pdf_floor(const double* quadratic, const double* eigenvalues, int F, int K, int T, int D,
                           double q_floor, double* quadratic_out, double* log_pdf, void* stream);

/* The log normalisers of ComplexWatson (complex_watson.py:89-214) for kappa (n), any values, dimension D
 * (0 < D <= 64), each formula in the reference's order of operations:
 *   PBB_CW_NORM_1F1     log_norm_1f1 (:157-168) = the mixture model's cw_log_norm: the series of 1F1(1; D; kappa)
 *                       below kappa = 20, Mardia's closed form above; finite where scipy's hyp1f1 overflows
 *                       (kappa > ~710), where the reference returns inf;
 *   PBB_CW_NORM_LOW     log_norm_low_concentration (:90-107), 20 Taylor terms;
 *   PBB_CW_NORM_MEDIUM  log_norm_medium_concentration (:110-138), kappa < 1e-2 clamped to 1e-2;
 *   PBB_CW_NORM_HIGH    log_norm_high_concentration (:141-154);
 *   PBB_CW_NORM_TRAN_VU log_norm_tran_vu (:171-214): low below kappa = 1 / D, the unclamped medium formula from
 *                       there on. */
enum { PBB_CW_NORM_1F1 = 0, PBB_CW_NORM_LOW = 1, PBB_CW_NORM_MEDIUM = 2, PBB_CW_NORM_HIGH = 3,
       PBB_CW_NORM_TRAN_VU = 4 };
int pbb_cw_log_norm(const double* kappa, long long n, int D, int variant, double* log_norm, void* stream);

/* ComplexWatson.log_pdf (complex_watson.py:73-87): log_pdf (M, N) = kappa |sum_d y_d conj(mode_d)|^2 -
 * log_norm_1f1(kappa, D) for y (M, N, D) as given (not normalised), mode (M, D) complex128, concentration (M).
 * 0 < D <= 64. */
int pbb_cw_log_pdf(const void* y, int dtype, long long y_stride, int M, int N, int D, const void* mode,
                   const double* concentration, double* log_pdf, void* stream);

/* Scratch of pbb_ccsg_log_pdf / pbb_ccsg_sample for M models (classes) of dimension D. */
size_t pbb_ccsg_workspace_bytes(int M, int D);

/* ComplexCircularSymmetricGaussian.log_pdf (complex_circular_symmetric_gaussian.py:26-48): log_pdf (M, N) =
 * -D log pi - log|det S| - Re(y^H S^-1 y) for y (M, N, D) and any invertible covariance S (M, D, D) complex128 --
 * np.linalg.slogdet and np.linalg.solve, not a Cholesky factor: one LU factorisation with partial pivoting per model
 * (a warp each), then one thread per (model, frame), so one model with many frames fills the GPU.  0 < D <= 64.
 * *status (reset by the call) = 1 + the first model with an exactly zero pivot (np.linalg.solve raises
 * LinAlgError); non-finite covariances give NaN, as in LAPACK. */
int pbb_ccsg_log_pdf(const void* y, int dtype, long long y_stride, int M, int N, int D, const void* covariance,
                     double* log_pdf, void* workspace, size_t workspace_bytes, int* status, void* stream);

/* ComplexCircularSymmetricGaussian.sample (:50-72) and sample_complex_angular_central_gaussian
 * (complex_angular_central_gaussian.py:58-65) for C classes at once; the standard normals are drawn on the host
 * (NumPy's global stream, in the reference's call order).  eigenvalues == NULL: a (C, D, D) are the covariances
 * (lower triangles read, like np.linalg.cholesky); else a are eigenvectors (columns) and the covariance is
 * V diag(eigenvalues) V^H (ComplexAngularCentralGaussian.covariance, :140-148).  normals (2, S, D): the real parts
 * of all S samples, then the imaginary parts; sample i belongs to the class c with offsets[c] <= i < offsets[c + 1]
 * (offsets (C + 1), offsets[0] = 0, offsets[C] = S) and is written to out row dest[i] (dest may be NULL: row i).
 * out (S, D) = L (re + i im) / sqrt(2), L = cholesky(covariance); unit_norm != 0 then divides every row by its
 * norm.  0 < D <= 64.  *status (reset by the call) = 1 + the first class whose covariance is not positive definite
 * (np.linalg.cholesky raises LinAlgError). */
int pbb_ccsg_sample(const void* a, const double* eigenvalues, int C, int D, const double* normals,
                    const long long* offsets, const long long* dest, long long S, int unit_norm, void* out,
                    void* workspace, size_t workspace_bytes, int* status, void* stream);

/* ComplexCircularSymmetricGaussianTrainer._fit, covariance_type 'full' (:94-116): covariance (F, D, D) =
 * sum_n s_n y_n y_n^H / max(sum_n s_n, denominator_floor) for observation (F, D, N) and saliency (F, N), or the
 * plain average over N without a saliency.  denominator_floor = np.finfo(y.dtype).tiny, the reference's floor (the
 * float32 tiny for complex64 y).  The sums are pbb_power_spectral_density's; N > 0, D < 35; workspace:
 * pbb_psd_workspace_bytes(F, N, D, 1). */
int pbb_ccsg_fit(const void* observation, int dtype, int F, int D, int N, const double* saliency,
                 double denominator_floor, void* covariance, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Building blocks of pb_bss.distribution.mixture_model_utils, pb_bss.distribution.utils, pb_bss.utils and
 * pb_bss.evaluation.sxr_module, csrc/api_mm_utils.cu.
 *
 * The operands are read and written in their own layouts: a pbb_nd_layout describes an index space (row-major over
 * `shape`) and, for every operand, the stride of every dim in elements (complex elements counted once); a stride of
 * 0 broadcasts the operand along that dim.  The arithmetic is fp64 and every result is rounded once to its storage
 * type; all sums run in a fixed order, so results are bit-reproducible from call to call.  Element types are PBB_F32,
 * PBB_F64, PBB_C64, PBB_C128 and, where stated, PBB_I32 / PBB_I64. */
#define PBB_ND_MAX_DIMS 8
#define PBB_ND_OPERANDS 4

typedef struct pbb_nd_layout {
  int nd; /* 0 <= nd <= PBB_ND_MAX_DIMS; nd = 0 is a single index */
  int reserved;
  long long shape[PBB_ND_MAX_DIMS];
  long long stride[PBB_ND_OPERANDS][PBB_ND_MAX_DIMS];
} pbb_nd_layout;

/* log_pdf_to_affiliation (mixture_model_utils.py:7-55) for any K: for every index c of `columns` (the dims of
 * log_pdf other than the class axis; operands 0 log_pdf, 1 weight, 2 mask, 3 out) and with class_stride[4] the
 * strides of the class axis of the same operands: a_k = exp(l_k - max_k l_k) * weight_k * mask_k, out_k =
 * a_k / max(sum_k a_k, tiny of dtype), clipped to [eps, 1 - eps] if eps != 0.  log_pdf and out are PBB_F32 / PBB_F64
 * (`dtype`), weight float64 (null: 1), mask bool bytes (null: all set). */
int pbb_affiliation_nd(const void* log_pdf, int dtype, const double* weight, const uint8_t* mask,
                       const pbb_nd_layout* columns, int K, const long long* class_stride, double affiliation_eps,
                       void* out, void* stream);

/* The reductions below cut the reduced index space of every output into chunks whose length depends on the number of
 * outputs and of reduced elements only -- about 16384 warps in all, at least 256 elements per chunk, one chunk when
 * the outputs alone are that many; a warp reduces one (output, chunk) -- lane l takes the elements l, l + 32, ... of the chunk in order, and
 * the lanes are combined by a fixed butterfly; fewer than 32 elements are one thread's loop -- and a second kernel
 * combines the chunk partials of every output in chunk order the same way.  The partition depends on the shapes only,
 * so results are bit-reproducible, and a long reduction with few outputs (np.sum over every axis, the frequency-tied
 * mixture weights) spreads over the whole GPU.  workspace: pbb_reduce_workspace_bytes(outputs, n) bytes, n = the
 * number of reduced elements per output. */
size_t pbb_reduce_workspace_bytes(long long outs, long long n);

/* The sum over a set of axes (np.sum / np.mean, estimate_mixture_weight mixture_model_utils.py:185-201, get_energy
 * sxr_module.py:13-14): for every index o of `outer` (operands 0 x, 1 multiplier, 2 out) the sum over the index space
 * `reduced` (operands 0 x, 1 multiplier) of v = x * multiplier (square = 0, real x) or v = re*re + im*im (square = 1,
 * no FMA), divided by `divisor`.  multiplier float64, may be null.  out is PBB_F32 or PBB_F64 (`out_dtype`). */
int pbb_axis_sum(const void* x, int dtype, const double* multiplier, const pbb_nd_layout* outer,
                 const pbb_nd_layout* reduced, int square, double divisor, void* out, int out_dtype, void* workspace,
                 size_t workspace_bytes, void* stream);

/* _unit_norm (pb_bss/distribution/utils.py:223-256): for every index r of `rows` (operands 0 x, 1 out; rows.nd < 8)
 * the vector norm of the n elements x_stride apart with np.linalg.norm's `ord` (2: sqrt of sum re*re + im*im; 1: sum
 * |x|; +inf / -inf: max / min |x|; 0: count of non-zeros; other p: (sum |x|^p)^(1/p)), then eps_style 0 'plus' (norm
 * + eps), 1 'max' (max(norm, eps)), 2 'where' (eps where norm == 0); then out = x / norm (out_stride apart; complex:
 * both parts divided) in a second pass over every element.  x and out have the same dtype; the norms are kept in the
 * workspace, pbb_reduce_workspace_bytes(rows, n). */
int pbb_unit_norm(const void* x, int dtype, const pbb_nd_layout* rows, long long n, long long x_stride,
                  long long out_stride, double ord, double eps, int eps_style, void* out, void* workspace,
                  size_t workspace_bytes, void* stream);

/* force_hermitian (pb_bss/distribution/utils.py:318-330): out = (A + A^H) / 2 of each of the `batch` contiguous
 * D x D matrices; real input stays real (A + A^T) / 2. */
int pbb_force_hermitian(const void* a, int dtype, long long batch, int D, void* out, void* stream);

/* abs_square (pb_bss/utils.py:314-336): out = re*re + im*im (complex, in the precision of the input, no FMA) or
 * x*x (real; PBB_I32 / PBB_I64 wrap like NumPy) of n contiguous elements; out has the real type of x. */
int pbb_abs_square(const void* x, int dtype, long long n, void* out, void* stream);

/* labels_to_one_hot (pb_bss/utils.py:234-311) written in its final layout: out (outer, C, inner) of elements of
 * elem_size bytes (1, 2, 4, 8 or 16) gets the bit pattern `one` (elem_size bytes, host pointer) where
 * labels[o][i] (int64, (outer, inner)) wraps to c (a negative label l counts as C + l), else zero bytes.  A label
 * outside [-C, C) sets *status (reset by the call) = 1 + its index (the smallest such index). */
int pbb_labels_to_one_hot(const long long* labels, long long outer, long long inner, int C, int elem_size,
                          const void* one, void* out, int* status, void* stream);

/* N *= factor of set_snr (sxr_module.py:51-78): out = x * factor over the index space `layout` (operands 0 x,
 * 1 factor (float64), 2 out); x and out of `dtype` (complex: both parts scaled), out may be x. */
int pbb_scale_nd(const void* x, int dtype, const double* factor, const pbb_nd_layout* layout, void* out,
                 void* stream);

/* VonMisesFisher.pdf (von_mises_fisher.py:82-83): exp of pbb_vmf_log_pdf, same arguments, in one pass. */
int pbb_vmf_pdf(const double* embedding, const double* mean, const double* concentration, const double* log_norm,
                int B, int N, int E, int K, double* pdf, void* stream);

/* ---- WPE dereverberation (nara_wpe.wpe; contract restated in oracle/wpe_oracle.py) -------------------------------
 * y is `bins` independent (D, T) problems of complex `dtype` (PBB_C64 / PBB_C128), element (b, d, t) at
 * b ysb + d ysd + t yst (element strides, any sign); out likewise with its own strides.  All arithmetic is fp64;
 * complex64 input is read as it is and the output rounded once at the store. */
#define PBB_WPE_MAX_N 96          /* taps * D */
#define PBB_WPE_MAX_D 30          /* channels: the per-bin solve, lstsq and filter kernels keep n x D blocks in
                                     shared memory, which fits the 227 KB of a CTA for every taps * D <= 96 up to here */
#define PBB_WPE_MAX_GROUP 65535   /* bins per group of pbb_wpe */
#define PBB_WPE_NONFINITE 1       /* status bit: a non-finite output value (e.g. an all-zero bin) */
#define PBB_WPE_LSTSQ 2           /* status bit: a bin's R had an exactly zero pivot and took the lstsq solution */

/* Workspace of pbb_wpe for `group` bins: the weights, the power scratch, the partial statistics, the filters and the
 * per-bin lstsq flags.  0 for an invalid shape. */
size_t pbb_wpe_workspace_bytes(long long group, int D, long long T, int taps, int delay, int valid);

/* wpe / wpe_v8 of nara_wpe.wpe: `iterations` times w = get_power_inverse(X, psd_context) per bin,
 * R = sum_S w_t Yt_t Yt_t^H, P = sum_S w_t Yt_t Y_t^H (Yt: build_y_tilde(Y, taps, delay); S every frame, or
 * t >= delay + taps - 1 with valid != 0), G = stable_solve(R, P) (np.linalg.solve; np.linalg.lstsq's minimum-norm
 * solution for a bin with an exactly zero pivot), X = Y - G^H Yt; iterations = 0 copies y.  psd_context < 0 means
 * inf.  out may be y (in place).  The bins run in groups of `group` bins sharing the workspace.  *status (reset by
 * the call) ORs PBB_WPE_NONFINITE and PBB_WPE_LSTSQ over all bins and iterations; read it after the stream. */
int pbb_wpe(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd, long long yst,
            void* out, long long osb, long long osd, long long ost, int taps, int delay, int iterations,
            long long psd_context, int valid, long long group, void* workspace, size_t workspace_bytes, int* status,
            void* stream);

/* pbb_wpe that also keeps, per iteration i < iterations, the filter G_i in G_save (iterations, bins, n, D)
 * complex128 and the weights w_i in w_save (iterations, bins, T) float64, both contiguous (both null: pbb_wpe).  The
 * launches and so the output are those of pbb_wpe; the copies are device-to-device on the stream. */
int pbb_wpe_forward(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                    long long yst, void* out, long long osb, long long osd, long long ost, int taps, int delay,
                    int iterations, long long psd_context, int valid, long long group, void* workspace,
                    size_t workspace_bytes, int* status, void* G_save, double* w_save, void* stream);

/* One WPE step with the caller's weights: R, P, G and X = Y - G^H Yt of pbb_wpe with w_t = weight[b wsb + t wst]
 * (float64, element strides) in place of the power.  Workspace pbb_wpe_workspace_bytes; G_out (null: not kept)
 * receives G (bins, n, D) complex128; *status as pbb_wpe. */
int pbb_wpe_step(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                 long long yst, const double* weight, long long wsb, long long wst, void* out, long long osb,
                 long long osd, long long ost, int taps, int delay, int valid, long long group, void* workspace,
                 size_t workspace_bytes, int* status, void* G_out, void* stream);

/* Backward of one WPE step, in torch's convention (the gradient of a real loss L is dL/dRe + i dL/dIm).  Per bin,
 * n = taps D, yt_t the delayed stack (row k D + d is y_{d, t - delay - k}), m_t = 1 for t in S (else 0), the forward
 * G = R^-1 P and x_t = y_t - G^H yt_t, and the incoming gradient xbar_t:
 *   Gbar = -sum_t yt_t xbar_t^H (every frame); R Pbar = Gbar with the forward's pivots (R is Hermitian, so the
 *     gradient of P is Pbar and that of R is -Pbar G^H);
 *   c_t = Pbar^H yt_t, u_t = xbar_t + m_t w_t c_t, b_t = m_t w_t x_t;
 *   ytbar_t = -G u_t + Pbar b_t (the R and P terms fold together through G^H yt_t = y_t - x_t);
 *   ybar_t = u_t + sum_k ytbar_{k D + d, t + delay + k} (the shift-add of ytbar onto y, a gather);
 *   wbar_t = m_t Re(c_t^H x_t).
 * An empty S (valid, T <= delay + taps - 1) makes G = 0 for every input: ybar = xbar, wbar = 0.
 * y as in pbb_wpe; weight (bins, T) float64 and G (bins, n, D) complex128 are the forward's (contiguous); xbar and
 * ybar (bins, D, T) complex128 contiguous, ybar accumulated (+=); wbar (bins, T) float64 written.  R is recomputed
 * with the forward's kernel and weights, so it is bit for bit the forward's.  A bin whose R has an exactly zero pivot
 * (the forward took lstsq) or is not finite gets NaN gradients; other bins are unaffected. */
size_t pbb_wpe_backward_workspace_bytes(long long group, int D, long long T, int taps, int delay, int valid);
int pbb_wpe_backward(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                     long long yst, const double* weight, const void* G, const void* xbar, int taps, int delay,
                     int valid, void* ybar, double* wbar, long long group, void* workspace, size_t workspace_bytes,
                     void* stream);

/* Backward of the power chain lambda_t = mean_d |x_dt|^2, lambda_c = its psd_context mean over the frames that exist
 * (psd_context < 0: inf), with x = y - G^H Yt (G (bins, taps D, D) complex128; null: x = y, taps and delay unused).
 * mode PBB_WPE_GRAD_PLAIN: gin (bins, T) is lambda_c's gradient (get_power).  PBB_WPE_GRAD_INVERSE: gin is the
 * gradient of w = 1 / max(lambda_c, 1e-10 M) with M the max per bin (wpe's weights); PBB_WPE_GRAD_INVERSE_ALL: the same
 * with M the max over all bins (get_power_inverse).  With z = max(lambda_c, eps M): zbar = -wbar / z^2, split as
 * torch.maximum does (all of it to the larger operand, half each on a tie); M's gradient eps sum(...) goes to the
 * maxima of lambda_c in equal shares (amax).  Then lambdabar_t = sum_{s : |s - t| <= c} lambdabar_c,s / n_s with n_s
 * the frames in s's window, and xbar_dt += (2 / D) lambdabar_t x_dt (xbar (bins, D, T) complex128 contiguous,
 * accumulated).  lambda_c is recomputed with the forward's kernel, so the max and its ties are the forward's. */
#define PBB_WPE_GRAD_INVERSE 0
#define PBB_WPE_GRAD_PLAIN 1
#define PBB_WPE_GRAD_INVERSE_ALL 2
size_t pbb_wpe_power_backward_workspace_bytes(long long bins, long long T);
int pbb_wpe_power_backward(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                           long long yst, const void* G, int taps, int delay, long long psd_context, int mode,
                           const double* gin, void* xbar, void* workspace, size_t workspace_bytes, void* stream);

/* Workspace of pbb_wpe_power: bins * T doubles. */
size_t pbb_wpe_power_workspace_bytes(long long bins, long long T);

/* get_power (inverse = 0) / get_power_inverse (inverse = 1) of nara_wpe.wpe, D <= PBB_WPE_MAX_D, any number of bins
 * below 2^31: out (bins, T) float64 contiguous,
 * lambda_t = mean over D of |y_dt|^2 with the psd_context moving mean (frames that exist only; < 0: the mean over all
 * frames); the inverse is 1 / max(lambda, 1e-10 max lambda), the max over all bins. */
int pbb_wpe_power(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                  long long yst, long long psd_context, int inverse, double* out, void* workspace,
                  size_t workspace_bytes, void* stream);

/* build_y_tilde of nara_wpe.wpe: out (bins, taps D, T) contiguous of y's dtype, row k D + d at frame t is
 * y_{d, t - delay - k}, zero where t - delay - k < 0. */
int pbb_wpe_build_y_tilde(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                          long long yst, int taps, int delay, void* out, void* stream);

/* ---- Frame-online WPE (nara_wpe.wpe.online_wpe_step; contract restated in oracle/wpe_online_oracle.py) -------
 * The recursive least-squares form of WPE (Yoshioka & Nakatani, IEEE TASLP 20(10), 2012; Caroselli et al.,
 * Interspeech 2017), one recursion per bin, n = taps D.  For frame t the window w (n) holds the frames
 * t - delay - 1 - k (k < taps) at index d taps + k, and one step is
 *   pred = y_t - G^H w, u = Q w, den = alpha lambda + w^H u, k = u / den, Q <- (Q - k (w^H Q)) / alpha,
 *   G <- G + k pred^H,
 * the division by alpha taken as a multiplication by 1 / alpha (exact for alpha = 1). */
#define PBB_WPE_ONLINE_MAX_SMEM 232448  /* bytes: pbb_wpe_online_smem_bytes must not exceed this (227 KB) */

/* Shared memory of one pbb_wpe_online CTA; taps + delay + 1 frames of D channels stay in it.  0 for an invalid
 * shape. */
size_t pbb_wpe_online_smem_bytes(int D, int taps, int delay);

/* online_wpe_step of nara_wpe.wpe over T >= 0 frames in one launch.  y: T frames of `bins` bins, element (b, d, t)
 * at b ysb + d ysd + t yst, complex `dtype`; history: the taps + delay frames before them, same dtype, own strides
 * (null: zeros).  power: null, or (bins) float64 lambda of the only frame (T = 1, the step API); when null, lambda
 * of frame t is the mean of |.|^2 over the D channels and the taps + delay + 1 frames t - taps - delay .. t,
 * history included, recomputed per frame in a fixed order.  inv_cov (bins, n, n) and filter_taps (bins, n, D)
 * complex128 row-major (null: identity, zeros); inv_cov_out and filter_taps_out receive Q and G after the last
 * frame (they may be the inputs).  z (b, d, t) gets pred of every frame, in y's dtype.  fp64 arithmetic, fixed-order
 * sums: a stream split over several calls (history and Q, G passed on) is bitwise equal to one call.  An all-zero
 * bin gives NaN in that bin. */
int pbb_wpe_online(const void* y, int dtype, long long bins, int D, long long T, long long ysb, long long ysd,
                   long long yst, const void* history, long long hsb, long long hsd, long long hst,
                   const double* power, const void* inv_cov, const void* filter_taps, void* z, long long zsb,
                   long long zsd, long long zst, void* inv_cov_out, void* filter_taps_out, int taps, int delay,
                   double alpha, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PBB_H_ */
