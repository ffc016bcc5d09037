/*
 * dfq_b200.h  -  C ABI of libdfq_sm90.so: the H100 (sm_90a) implementation of the data-free
 * quantization calibration hot path of jakc4103/DFQ.
 *
 * The reference is pure Python on PyTorch-eager CPU tensors and has NO foreign-function interface
 * of its own (SURVEY.md section 2.1); each entry point below therefore cites the reference Python
 * function (file:line under /root/reference) whose arithmetic it replaces.  A maintainer binds them
 * with ctypes exactly as dfq_b200/_lib.py does; INTEGRATION.md shows the stub.
 *
 * Conventions
 *   - plain C: pointers + sizes, no torch / C++ types.  All tensor pointers are DEVICE pointers to
 *     fp32 owned by the caller; descriptor tables (DfqLayer, DfqRelation, ...) are HOST pointers and
 *     are copied to the device by the call.
 *   - every function returns 0 on success, a positive cudaError_t or a negative DFQ_E_* code;
 *     dfq_last_error() returns a human readable message for the calling thread.
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it.  Functions that
 *     return results to host memory (marked "synchronises") wait for the stream.
 *   - nothing is allocated that the caller can see; scratch is carved from caller-provided arenas
 *     or from a per-process workspace that the library owns.
 */
#ifndef DFQ_B200_H_
#define DFQ_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DFQ_ABI_VERSION 6

enum {
  DFQ_OK = 0,
  DFQ_E_ARG = -1,        /* invalid argument (null pointer, bad size, inconsistent descriptor) */
  DFQ_E_UNSUPPORTED = -2,
  DFQ_E_NOT_COOPERATIVE = -3 /* device cannot co-schedule the persistent grid */
};

/* ---------------------------------------------------------------------------------------------
 * library / device
 * ------------------------------------------------------------------------------------------- */
int dfq_abi_version(void);
const char* dfq_last_error(void);
/* sizeof() of the descriptor structs as compiled (0 DfqLayer, 1 DfqRelation, 2 DfqCleParams,
 * 3 DfqCleResult, 4 DfqFold, 5 DfqExpectTerm, 6 DfqBcLayer, 7 DfqQuantTask, 8 DfqI8Conv, 9 DfqI8Epilogue): lets a binding verify
 * its struct mirrors without a GPU. */
int dfq_struct_size(int which);
/* number of SMs and max co-resident CTAs of the persistent kernels on the current device */
int dfq_device_info(int* sm_count, int* engine_ctas);

/* ---------------------------------------------------------------------------------------------
 * The calibration arena
 *
 * All weights, biases and per-channel vectors of one model (or of one rank's shard of it) live in a
 * single fp32 device buffer, the "arena".  Descriptors address it by float offsets.  Weight offsets
 * are multiples of 4 floats (16 B) so rows of length % 4 == 0 can be moved with 128-bit accesses.
 * ------------------------------------------------------------------------------------------- */

/* One target layer: Conv2d weight [rows, cols, k, k] (kk = k*k) or Linear weight [rows, cols] (kk=1),
 * row-major contiguous, i.e. `rows` rows of row_len = cols*kk floats.  cols = in_channels / groups. */
typedef struct DfqLayer {
  int64_t w_off;      /* weight                                                          */
  int64_t bias_off;   /* bias[rows]; every layer on the path owns one (zeros if the module had none,
                         dfq.py:91-92, layer_transform.py:253-254)                         */
  int32_t rows;
  int32_t cols;
  int32_t kk;
  int32_t rel_in;     /* relation in which this layer is `second` (its columns get 1/s), or -1 */
  int32_t rel_out;    /* relation in which this layer is `first`  (its rows get s),      or -1 */
  int32_t col_mode;   /* how the column ranges needed by rel_in are kept current between sweeps:
                         0 = chain end: only column-scaled  -> ranges updated analytically
                         1 = depthwise middle (cols==1, one row per group) -> analytic as well
                         2 = general middle layer -> re-scanned after its pass               */
  int32_t group;      /* convergence group (= model) this layer belongs to, 0 .. n_groups-1    */
  int32_t flags;      /* DFQ_LAYER_COLS_READY: buffer 0 of cmin/cmax already holds the column extrema of the
                         current weights (dfq_bn_fold with DfqFold.scan_go > 0 just produced them): dfq_cle_run
                         skips its initial scan of this layer
                         DFQ_LAYER_FOLD_PENDING: see below                                     */
  int64_t cmin_off;   /* [2][C of rel_in] running column minima, double-buffered by sweep parity
                         (scratch, valid when rel_in >= 0)                                  */
  int64_t cmax_off;   /* [2][C of rel_in] running column maxima                              */
  int64_t fold_off;   /* DFQ_LAYER_FOLD_PENDING: [rows] fold factors gamma/sqrt(var+eps) (DfqFold.fac_off)      */
} DfqLayer;

/* Both flags are promises about the call that runs RIGHT AFTER dfq_bn_fold, on the same weights:
 *   DFQ_LAYER_COLS_READY   the fold (scan_go > 0) has written buffer 0 of the column extrema of the FOLDED weights.
 *   DFQ_LAYER_FOLD_PENDING the fold ran with DfqFold.mode = DFQ_FOLD_DEFER: biases, BN vectors and the factors at fold_off
 *                          are final, the weights are NOT yet multiplied by the factors.  dfq_cle_run completes the fold:
 *                          k_cle_stack multiplies each row by its factor as its first sweep reads it (fl(w * f), the value
 *                          the fold would have stored); on every other path (the engine, no sweep at all) the fold is
 *                          applied to the weights before anything else.  Either way the weights are folded on return. */
#define DFQ_LAYER_COLS_READY 1
#define DFQ_LAYER_FOLD_PENDING 2

/* One equalization relation (utils/relation.py:5-27): rows of `first` are multiplied by s[c],
 * the matching input columns of `second` by 1/s[c] (dfq.py:62-73). */

typedef struct DfqRelation {
  int32_t first;
  int32_t second;
  int32_t channels;   /* C1 = rows of first                                   */
  int32_t groups;     /* G  = 1 if C1 == cols(second) else C1 / cols(second)  (dfq.py:29-32) */
  int32_t gi;         /* C1 / G                                               */
  int32_t go;         /* rows(second) / G                                     */
  int64_t bn_w_off;   /* BN fake_weight[C1] scaled with the rows (dfq.py:64-65), or -1 */
  int64_t bn_b_off;   /* BN fake_bias[C1]                        (dfq.py:67-68), or -1 */
  int64_t s_acc_off;  /* [C1] accumulated product of per-sweep s = Relation.S (relation.py:20-24) */
  int64_t s_step_off; /* [C1] scratch: s of the current sweep          */
  int64_t inv_off;    /* [C1] scratch: the reciprocal applied to the columns this sweep */
} DfqRelation;

typedef struct DfqCleParams {
  float s_lo, s_hi;        /* s_range, already rounded to fp32 (comparisons are fp32, dfq.py:59) */
  float inv_lo, inv_hi;    /* fp32(1.0/s_lo), fp32(1.0/s_hi): reciprocal of a clamped s (dfq.py:73) */
  float eps;               /* dfq.py:58 */
  int32_t signed_mode;     /* 0: range = max-min (dfq.py:54-55), 1: range = max|w| (dfq.py:50-51) */
  double converge_thres;   /* dfq.py:78 */
  int32_t converge_count;
  int32_t max_sweeps;      /* >0: stop after this many sweeps regardless (1 = one _layer_equalization pass) */
  int32_t apply_only;      /* 1: do not solve - take s from s_acc (a scale vector computed elsewhere) and apply it:
                              rows of `first` *= S, columns of `second` *= 1/S.  Use with max_sweeps = 1. */
  int32_t _pad;
} DfqCleParams;

typedef struct DfqCleResult {
  int32_t n_sweeps;
  int32_t converged;       /* exit rule of dfq.py:83 fired (as opposed to max_sweeps)            */
  double last_diff;        /* `diff` of dfq.py:110 at exit                                        */
  double diffs[64];        /* diff_tmp of the first 64 sweeps (dfq.py:105-108)                    */
} DfqCleResult;

/* Cross-layer equalization to convergence.  Replaces dfq.py:78-117 (cross_layer_equalization) and,
 * with max_sweeps = 1 and a single relation, dfq.py:28-75 (_layer_equalization).
 *
 * `steps` partitions the layers touched by the relations by chain position: step_ptr[n_steps+1]
 * indexes step_layers[]; step p holds the p-th layer of every chain.  Relations must be listed in
 * forward chain order (every layer's rel_in precedes its rel_out in `rels`), which is the order
 * utils/relation.py:61-68 produces.  One persistent cooperative kernel runs all sweeps; the exit
 * rule of dfq.py:105-115 is evaluated on the device; the convergence metric sums mean|W - W_prev|
 * over the layers listed in the steps (layers outside every relation never change, so their term of
 * dfq.py:105-108 is zero).  Synchronises (result is read back).
 *
 * Convergence groups.  The reference calibrates ONE model per call, and its exit rule sums over that model's
 * layers.  A batch of independent models (e.g. the synthetic stack of BASELINE.json, whose blocks are independent
 * two-layer models) is passed as n_groups > 1 with DfqLayer.group naming the model of each layer: every group is
 * iterated until ITS exit rule fires - exactly what one reference call per model would do - while all groups
 * share the launch.  result->n_sweeps is the maximum over groups, ->converged the conjunction, ->diffs and
 * ->last_diff belong to group 0. */
int dfq_cle_run(float* arena, int64_t arena_floats,
                const DfqLayer* layers, int32_t n_layers,
                const DfqRelation* rels, int32_t n_rels,
                const int32_t* step_ptr, const int32_t* step_layers, int32_t n_steps,
                const DfqCleParams* params, DfqCleResult* result,
                int32_t n_groups, int32_t* group_sweeps /* host, [n_groups] sweeps run per group, or NULL */,
                void* stream);

/* *takes = 1 when dfq_cle_run would run this problem (same tables, DfqCleParams.apply_only = apply_only) on the
 * streaming stack kernel k_cle_stack on the current device, 0 when on k_cle_engine - the one decision dfq_cle_run makes
 * (including the DFQ_CLE_STACK override).  A fold may defer its weight pass (DFQ_FOLD_DEFER) only into a k_cle_stack run:
 * on the engine path the deferred fold costs an extra pass.  No GPU work, no synchronisation. */
int dfq_cle_takes_stack(const DfqLayer* layers, int32_t n_layers, const DfqRelation* rels, int32_t n_rels,
                        const int32_t* step_ptr, const int32_t* step_layers, int32_t n_steps, int32_t apply_only,
                        int32_t* takes);

/* BN fold (utils/layer_transform.py:231-276, merge_batchnorm), batched over layers.
 * W[o,:] *= gamma[o]/sqrt(var[o]+eps); b = b*f + (beta - gamma*mean/sqrt(var+eps));
 * fake_weight = |gamma|, fake_bias = beta. */
typedef struct DfqFold {
  int32_t layer;
  float bn_eps;
  int64_t gamma_off, beta_off, mean_off, var_off;   /* inputs  [rows] */
  int64_t fake_w_off, fake_b_off;                   /* outputs [rows] */
  int32_t scan_go, scan_gi;   /* > 0: the layer is `second` of a relation with `scan_go` rows and `scan_gi` columns per
                                 group (DfqRelation.go / .gi): also write the column extrema of the FOLDED weights into
                                 buffer 0 of the layer's cmin_off / cmax_off (layers[] must carry them), saving the
                                 equalization its initial 4 B/weight scan.  0: no scan. */
  int32_t mode;               /* DFQ_FOLD_FULL / _DEFER / _APPLY, below                                              */
  int32_t _pad;
  int64_t fac_off;            /* _DEFER, _APPLY: [rows] fold factors gamma/sqrt(var+eps)                              */
} DfqFold;
/* DFQ_FOLD_FULL   the fold above: weights, bias, fake_weight / fake_bias.
 * DFQ_FOLD_DEFER  everything but the weights: bias, fake_weight / fake_bias, and each row's factor into fac_off.  With
 *                 scan_go > 0 the weights are READ (not written) and the column extrema of fl(w * factor) - those of the
 *                 folded weights - go to buffer 0.  The weights stay unfolded until a DFQ_LAYER_FOLD_PENDING layer entry
 *                 (fold_off = fac_off) hands them to dfq_cle_run, or a DFQ_FOLD_APPLY call completes the fold.
 * DFQ_FOLD_APPLY  the weights only: W[o,:] = fl(W[o,:] * fac[o]); gamma / beta / mean / var / bias are not read. */
#define DFQ_FOLD_FULL 0
#define DFQ_FOLD_DEFER 1
#define DFQ_FOLD_APPLY 2
int dfq_bn_fold(float* arena, int64_t arena_floats, const DfqLayer* layers, int32_t n_layers,
                const DfqFold* folds, int32_t n_folds, void* stream);

/* Bias correction (dfq.py:173-293).  The host walks the graph (find_prev_bn, layer_transform.py:
 * 299-344) and emits, per corrected layer, the recipe of its input expectation: a list of terms,
 * each one BN (fake_weight/fake_bias offsets, `relu` flag) combined by concatenation or summation
 * (dfq.py:244-278).  The device evaluates E[x] (float64 pdf/cdf like scipy, dfq.py:182-184), the
 * 8-bit quantization error of the weights (dfq.py:216-219), the grouped mat-vec (dfq.py:281-287),
 * subtracts it from the bias (:292) and forwards -delta to the next BN's fake_bias (:204-206,293).
 * Layers are processed level by level; levels are separated by grid barriers. */
typedef struct DfqExpectTerm {
  int64_t bn_w_off, bn_b_off;
  int32_t n;            /* BN channels */
  int32_t relu;         /* 1: rectified-Gaussian mean (dfq.py:238-240), 0: fake_bias (:242) */
  int32_t dst_off;      /* where this term lands in the layer's expectation vector (cat: running
                           offset, add: offset of the accumulator it is added to)          */
  int32_t accumulate;   /* 0: store, 1: add (dfq.py:270) */
} DfqExpectTerm;

typedef struct DfqBcLayer {
  int32_t layer;
  int32_t signed_mode;       /* symmetric quantizer (dfq.py:218) */
  int32_t term_begin, term_end;  /* into terms[] */
  int32_t expect_len;        /* = groups * cols */
  int32_t flags;             /* bit 0: use sum_k W instead of the quantization error (bias absorption,
                                dfq.py:139-153); bit 1: ADD delta to the bias (dfq.py:164) instead of
                                subtracting it (dfq.py:292) */
  int64_t expect_off;        /* scratch [expect_len] */
  int64_t delta_off;         /* scratch/out [rows]: eps . E[x]                           */
  int64_t next_bn_b_off;     /* fake_bias that receives -delta (dfq.py:204-206), or -1  */
  int64_t minmax_off;        /* scratch [2]: per-tensor min/max of W                     */
  int64_t colmin_off;        /* n_col > 0: [n_col] column minima / maxima of the CURRENT weights that the caller vouches */
  int64_t colmax_off;        /* for; the per-tensor range (dfq.py:14) is reduced from them and the weights are not      */
  int32_t n_col;             /* streamed a second time.  After dfq_cle_run the valid buffer of a `second` layer is      */
  int32_t _pad;              /* cmin_off + (group_sweeps[group] & 1) * C (same for cmax).  0: scan the weights.          */
} DfqBcLayer;
int dfq_bias_correct(float* arena, int64_t arena_floats, const DfqLayer* layers, int32_t n_layers,
                     const DfqBcLayer* bc, int32_t n_bc, const DfqExpectTerm* terms, int32_t n_terms,
                     const int32_t* level_ptr, int32_t n_levels, int32_t num_bits, void* stream);

/* Per-tensor min/max + in-place fake quantization of arena tensors, batched
 * (utils/layer_transform.py:279-296 quantize_targ_layer; CPU semantics: true division). */
typedef struct DfqQuantTask {
  int64_t off;          /* tensor offset in the arena */
  int64_t n;
  int32_t num_bits;
  int32_t symmetric;
  int64_t minmax_off;   /* scratch [2] */
} DfqQuantTask;
int dfq_quantize_tensors(float* arena, int64_t arena_floats, const DfqQuantTask* tasks, int32_t n_tasks,
                         int div_mode /* 0: true division (CPU-resident params), 1: reciprocal (CUDA) */,
                         void* stream);

/* ---------------------------------------------------------------------------------------------
 * Stand-alone tensor kernels (activations, module forward, API-level helpers)
 * ------------------------------------------------------------------------------------------- */

/* out2[0] = min(x), out2[1] = max(x)   (dfq.py:14, layer_transform.py:289, quantize.py:195-196) */
int dfq_minmax(const float* x, int64_t n, float* out2, void* stream);

/* Fake quantization with explicit scalars (quantize.py:70-74); `scale` is the Python double of quantize.py:64-66:
 *   t = x + (-min);  t = div_mode ? t * fp32(1.0/scale) : t / fp32(scale);  t = clamp(t, qmin, qmax);
 *   t = rint(t) [-> codes, if non-null];  y = t * fp32(scale);  y = y + min_value.
 * Four separately rounded fp32 ops, no FMA contraction.  div_mode 0 = IEEE division (PyTorch CPU), 1 = multiply by
 * the reciprocal formed in double and rounded to fp32 - what PyTorch CUDA eager computes for `div_(python_float)`
 * [probed with torch 2.11].  y may alias x. */
int dfq_quant_dequant(const float* x, float* y, int64_t n, float min_value, double scale,
                      float qmin, float qmax, int div_mode, float* codes, void* stream);

/* Same with the range taken from device memory (*min_ptr, *max_ptr: e.g. the two halves of a dfq_minmax
 * result, or QuantMeasure's running_min / running_max buffers) and the scalar prologue of
 * quantize.py:49-66 evaluated on the device: no host synchronisation (replaces the float() syncs of
 * quantize.py:119,195-196).
 *   prologue 0: min/max widened to double, scale formed in double (the reference passed float(min),
 *               float(max): quantize.py:119,195-196, layer_transform.py:289, dfq.py:14)
 *   prologue 1: min/max are fp32 0-d tensors in the reference (min_value=None, quantize.py:24-35): scale
 *               formed by fp32 tensor ops, `/ (qmax-qmin)` a true division (CPU tensors)
 *   prologue 2: as 1 with `/ (qmax-qmin)` a multiply by the fp32 reciprocal (CUDA tensors)
 * With prologue 1/2 the element-wise division is by a tensor and therefore always a true division. */
int dfq_quant_dequant_dev(const float* x, float* y, int64_t n, const float* min_ptr, const float* max_ptr,
                          int num_bits, int symmetric, int div_mode, int prologue, float* codes, void* stream);

/* Observer statistics (quantize.py:106-107,110-111): out2[0] = mean_b min(x[b,:]),
 * out2[1] = mean_b max(x[b,:]) for x viewed as [batch, per_sample]. */
int dfq_act_minmax_per_sample(const float* x, int64_t batch, int64_t per_sample, float* out2,
                              float* scratch_2b /* [2*batch] */, void* stream);

/* QuantMeasure running statistics update on the device (quantize.py:103-113), stat2 = {min, max}:
 * mode 1: running_min = min(running_min, stat_min), running_max = max(running_max, stat_max)  (update_stat)
 * mode 2: running = running*(1-momentum) + stat*momentum                                      (training EMA) */
int dfq_observer_update(float* running_min, float* running_max, const float* stat2, int mode, double momentum,
                        void* stream);

/* QuantMeasure.forward in ONE launch (quantize.py:102-119; SURVEY 8(f) rank 1): per-sample min/max -> batch mean -> running
 * statistics update -> fake quantization of x into y, a persistent cooperative kernel with one grid barrier.  flags:
 *   DFQ_OBS_UPDATE (1)  update_stat: running = (min(running_min, stat_min), max(running_max, stat_max))  quantize.py:103-107
 *   DFQ_OBS_EMA    (2)  training: running = running*(1-momentum) + stat*momentum (after the update), and the range used for
 *                       quantization is the batch statistic                                               quantize.py:109-113
 *   DFQ_OBS_OWN    (4)  no running buffers (may be NULL): quantize with the statistic itself - with batch = 1 this is
 *                       quantize(w, bits, float(w.min()), float(w.max())) (quantize.py:194-196) or, with prologue 1/2, the
 *                       implicit-range path of quantize.py:24-35 used for biases
 * Without DFQ_OBS_EMA / DFQ_OBS_OWN the range is the updated running pair (quantize.py:115-119).  stat_out2 (optional)
 * receives the batch statistic.  div_mode / prologue as in dfq_quant_dequant_dev. */
#define DFQ_OBS_UPDATE 1
#define DFQ_OBS_EMA 2
#define DFQ_OBS_OWN 4
int dfq_observe_quant(const float* x, float* y, int64_t batch, int64_t per_sample, float* running_min, float* running_max,
                      float* stat_out2, int flags, double momentum, int num_bits, int symmetric, int div_mode, int prologue,
                      void* stream);

/* HOST-side helper of the residency (no CUDA call): copies n segments between scattered host buffers and one contiguous
 * staging image - what Session.upload()/download() do around their single H2D / D2H copy (the reference moves a model with
 * one `.cuda()` / `.cpu()` per tensor: main_cls.py:70, dfq.py:145-151).  Segment i is ptr[i] (host address), bytes[i] long and
 * lives at byte offset off[i] of `staging`.  dir 0: staging <- segments (gather), dir 1: segments <- staging (scatter).
 * threads <= 0: min(8, hardware threads); never more than one thread per MB. */
int dfq_host_copy_segments(void* staging, void* const* ptr, const size_t* bytes, const size_t* off, int n, int dir, int threads);

/* BN-statistics matching loss of the distilled-data generation (ZeroQ/distill_data.py:171-196; SURVEY 8(f) rank 2) on one
 * BatchNorm input x [n, c, hw] (contiguous):  loss2[0] = sum_{n,c} (bn_mean[c] - mean_hw x)^2 / c,
 * loss2[1] = sum_{n,c} (bn_std[c] - std_hw(x + eps))^2 / c  (unbiased std; own_loss, distill_data.py:41-46).
 * One pass over x; mean_out / std_out [n*c] are kept for the backward pass. */
int dfq_bnstat_loss_fwd(const float* x, int64_t n, int64_t c, int64_t hw, const float* bn_mean, const float* bn_std,
                        float eps, float* mean_out, float* std_out, double* loss2, void* stream);
/* d(g[0]*loss2[0] + g[1]*loss2[1]) / dx written (accumulate = 0) or added (1) to grad_x; grad_loss2 = device float[2]. */
int dfq_bnstat_loss_bwd(const float* x, float* grad_x, int64_t n, int64_t c, int64_t hw, const float* bn_mean,
                        const float* bn_std, float eps, const float* mean_in, const float* std_in,
                        const float* grad_loss2, int accumulate, void* stream);

/* Per-row extrema of a [rows, row_len] matrix (dfq.py:50,54: range of weight_first_group[ii]). */
int dfq_range_rows(const float* w, int64_t rows, int64_t row_len, float* out_min, float* out_max,
                   void* stream);

/* Per-input-column extrema of W[O, J, kk] within `groups` row groups (dfq.py:51,55: range of
 * weight_second_group[:, ii]); out arrays have groups*J entries. */
int dfq_range_cols(const float* w, int64_t O, int64_t J, int64_t kk, int64_t groups,
                   float* out_min, float* out_max, void* stream);

/* *out = mean |a - b| accumulated in double (dfq.py:108). */
int dfq_mean_abs_diff(const float* a, const float* b, int64_t n, double* out, void* stream);

/* Q(W) - W written to `eps` (dfq.py:8-25, reduction=None) for a tensor with known min/max. */
int dfq_quant_error(const float* w, float* eps, int64_t n, const float* minmax2, int num_bits,
                    int symmetric, void* stream);

/* Library self-test hook.  The streaming bias-correction kernel evaluates quantize.py:70-74 without division / rounding
 * instructions (Markstein-corrected reciprocal product, magic-number rint; dfq_b200/csrc/bc_stream.cuh) when a per-tensor
 * guard allows it.  This entry computes Q(w) - w of one tensor both ways: eps_fast with that arithmetic, eps_div with the
 * plain IEEE chain, *ok_dev = the guard's verdict for this tensor's (min, max).  The two arrays must be bit-identical
 * whenever *ok_dev == 1 (tests/test_gpu_engine.py). */
int dfq_selftest_bc_arithmetic(const float* w, float* eps_fast, float* eps_div, int64_t n, const float* minmax2,
                               int num_bits, int symmetric, int* ok_dev, void* stream);

/* x = clamp(x, lo, hi) in place (dfq.py:167-170 clip_weight). */
int dfq_clamp(float* x, int64_t n, float lo, float hi, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Int8 execution of calibrated layers
 *
 * The reference's "true int8 inference" writes the scales of convert_ncnn.py:178-201 into an ncnn table and lets ncnn's
 * runtime execute the model in int8 on a CPU (ncnn2int8, inference_cls.cpp).  These entries run the same dequantizing
 * int8 convolution on the H100, one layer at a time with fp32 NCHW in and out:
 *   q(v, s) = clamp(round_half_away(fp32(v * s)), -127, 127)    activations: one scale a; weights: w_s[o] per channel
 *   acc     = exact int32 sum of q(x) * q(w) over the receptive field (padding contributes 0)
 *   y       = fp32(fp32_rn(acc) * dq[o]) + bias[o],   dq[o] = fp32(1 / fp32(a * w_s[o]))  (computed by the caller)
 * Supported: groups == 1 (implicit GEMM on the tensor cores; Linear is the 1x1 case on [B, I, 1, 1]) and depthwise
 * groups == C == O (CUDA cores).  Any other grouping returns DFQ_E_UNSUPPORTED.
 * ------------------------------------------------------------------------------------------- */
typedef struct DfqI8Conv {
  int32_t N, C, H, W;          /* input [N, C, H, W]                                                           */
  int32_t O, kh, kw;           /* output channels, kernel size                                                 */
  int32_t stride_h, stride_w;
  int32_t pad_h, pad_w;        /* zero padding                                                                 */
  int32_t dil_h, dil_w;
  int32_t groups;
  int32_t OH, OW;              /* (H + 2 pad - dil (k - 1) - 1) / stride + 1, checked                          */
  int32_t Cpad;                /* channel stride of the int8 NHWC codes and packed weights: C rounded up to 16 */
  int32_t _pad;
} DfqI8Conv;

/* Activation quantizer: fp32 NCHW x -> int8 NHWC q[N, H, W, Cpad], pad channels 0.  q must be 16-byte aligned. */
int dfq_i8_quantize_nhwc(const float* x, int8_t* q, int32_t N, int32_t C, int32_t H, int32_t W, int32_t Cpad, float scale,
                         void* stream);
/* Weight packer (once per layer, at conversion): fp32 w[O, C/groups, kh, kw] with per-output-channel scales w_scale[O]
 * -> groups == 1: int8 [O][kh][kw][Cpad]; depthwise: int8 [kh*kw][Cpad].  Pad channels 0.  Uses g's O, C, kh, kw, groups, Cpad. */
int dfq_i8_pack_weights(const float* w, const float* w_scale, int8_t* packed, const DfqI8Conv* g, void* stream);
/* Convolution of quantized codes with the epilogue above: xq from dfq_i8_quantize_nhwc, wq from dfq_i8_pack_weights, dq[O],
 * bias[O] (NULL: none), y fp32 [N, O, OH, OW].  acc_out (NULL: not written) receives the int32 sums, [N, O, OH, OW]. */
int dfq_i8_conv(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, float* y, int32_t* acc_out,
                const DfqI8Conv* g, void* stream);
/* The same convolution with a requantizing epilogue, for two layers chained through int8 codes (ncnn's fused requantize):
 *   v  = fp32(fp32_rn(acc) * dq[o]) + bias[o]
 *   v  = v < act_lo ? act_lo : (v > act_hi ? act_hi : v)       the activation as one clamp; NaN stays NaN
 *   yq = q(v, out_scale)                                       out_scale: the NEXT layer's activation scale
 * yq is int8 NHWC [N, OH, OW, round_up(O, 16)], the layout dfq_i8_quantize_nhwc gives the next layer, whatever the input's
 * g->Cpad; pad channels are written 0 and nothing past them.  ReLU is (0, +inf), ReLU6 (0, 6), no activation (-inf, +inf).  yq must be 16-byte aligned; NaN or
 * unordered bounds and an out_scale that is not finite and non-negative are DFQ_E_ARG. */
int dfq_i8_conv_requant(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, int8_t* yq,
                        float out_scale, float act_lo, float act_hi, const DfqI8Conv* g, void* stream);

/* The residual epilogue of dfq_i8_conv_fused: the convolution, the pass-throughs up to a residual block's add, the add and
 * the pass-throughs after it, in one launch.  Per output element (n, o, p):
 *   v  = fp32(fp32_rn(acc) * dq[o]) + bias[o]
 *   v  = v < pre_lo ? pre_lo : (v > pre_hi ? pre_hi : v)       NaN stays NaN
 *   v  = fp32(v + residual[n, o, p])                           only when residual != NULL: fp32 NCHW [N, O, OH, OW]
 *   v  = v < post_lo ? post_lo : (v > post_hi ? post_hi : v)
 *   y[n, o, p]  = v                                            when y != NULL: fp32 NCHW [N, O, OH, OW]
 *   yq[n, p, o] = q(v, out_scale)                              when yq != NULL: int8 NHWC [N, OH, OW, round_up(O, 16)], as
 *                                                              dfq_i8_conv_requant writes it (pad channels 0)
 * No clamp is (-inf, +inf). */
typedef struct DfqI8Epilogue {
  const float* residual;
  float* y;
  int8_t* yq;
  float out_scale, pre_lo, pre_hi, post_lo, post_hi;
} DfqI8Epilogue;
/* The convolution of dfq_i8_conv with the epilogue *e.  DFQ_E_ARG, with a reason: y and yq both NULL, yq not 16-byte
 * aligned, residual or y not 4-byte aligned, NaN or unordered bounds in either clamp, an out_scale that is not finite and non-negative while yq is written,
 * a residual that overlaps y or yq, or y overlapping yq (extents from the geometry).  Grouping as dfq_i8_conv. */
int dfq_i8_conv_fused(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, const DfqI8Epilogue* e,
                      const DfqI8Conv* g, void* stream);

/* The convolution's codes written into a channel slice of a wider int8 NHWC tensor, for a channel concatenation whose
 * producers each write their own channels of the consumer's input:  pixel m, channel o < round_up(O, 16) goes to
 * e->yq[m * cstride + coff + o] (pad channels O .. round_up(O, 16) written 0; the last slice's are the tensor's pad), and
 * nothing else of e->yq is written.  The codes are those of dfq_i8_conv_fused with the epilogue *e (residual and y as
 * there; yq required); without residual and y and with post = (-inf, +inf), those of dfq_i8_conv_requant at
 * (out_scale, pre_lo, pre_hi).  coff = 0, cstride = round_up(O, 16) is the tensor those two entries write.  DFQ_E_ARG, with
 * a reason: yq NULL or not 16-byte aligned, coff or cstride not a multiple of 16, coff + round_up(O, 16) > cstride, a
 * residual or y that overlaps the slice's extent or each other, and the epilogue refusals of dfq_i8_conv_fused. */
int dfq_i8_conv_slice(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, const DfqI8Epilogue* e,
                      int32_t coff, int32_t cstride, const DfqI8Conv* g, void* stream);

/* Max pooling, with torch's geometry (F.max_pool2d: zero-free padding, dilation, ceil_mode). */
typedef struct DfqI8Pool {
  int32_t N, C, H, W;          /* input [N, C, H, W]                                                              */
  int32_t kh, kw;
  int32_t stride_h, stride_w;
  int32_t pad_h, pad_w;        /* at most kh / 2 and (dil_h (kh - 1) + 1) / 2, as torch requires                   */
  int32_t dil_h, dil_w;
  int32_t ceil_mode;           /* 0 or 1                                                                          */
  int32_t OH, OW;              /* torch's formula, checked; in ceil mode the last window starts inside the input   */
  int32_t Cpad;                /* channel stride of the codes: a multiple of 16 >= C                              */
} DfqI8Pool;
/* Two modes, by which input is given (exactly one):
 *   xq (codes): int8 NHWC [N, H, W, Cpad] -> yq int8 NHWC [N, OH, OW, Cpad], the byte-wise signed max of the taps inside
 *      the input.  q(v, s) is monotone for s >= 0, so this is q(max_pool2d(v), s) for any window without NaN.  Exceptions
 *      of the per-layer path, where it quantizes the fp32 max: a window holding a NaN gives -127 there and the max of the
 *      other codes here; at scale 0 an infinite input gives q(inf * 0) = -127 there.  A window with no tap in the input
 *      gives -127 (torch's -inf), pad channels 0.  y must be NULL.
 *   x (fp32): NCHW [N, C, H, W] -> y fp32 NCHW [N, C, OH, OW] (NULL: not written) bit for bit torch's CUDA max_pool2d (from
 *      -inf, taps row-major, replaced when v > max or v is NaN: the first of tied values, -0.0 before +0.0, is kept), and /
 *      or yq = q(y, out_scale) int8 NHWC [N, OH, OW, Cpad] (NULL: not written; pad channels 0).
 * DFQ_E_ARG, with a reason: a bad geometry, both or neither input, no output, misaligned xq / yq (16 B) or x / y (4 B),
 * an out_scale that is not finite and non-negative while yq is written in fp32 mode, overlapping input and outputs. */
int dfq_i8_maxpool(const int8_t* xq, const float* x, float* y, int8_t* yq, float out_scale, const DfqI8Pool* g,
                   void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DFQ_B200_H_ */
