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

#define DFQ_ABI_VERSION 11

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
 * 3 DfqCleResult, 4 DfqFold, 5 DfqExpectTerm, 6 DfqBcLayer, 7 DfqQuantTask, 8 DfqI8Conv, 9 DfqI8Epilogue, 10 DfqI8Pool,
 * 11 DfqI8Resize, 12 DfqI8Affine, 13 DfqI8AffineEpilogue, 14 DfqI8AffineObserve, 15 DfqI8AffineLayout,
 * 16 DfqI8AffineResize, 17 DfqI8AffineRows, 18 DfqSsdNms, 19 DfqSegArgmax, 21 DfqPreImage, 22 DfqPreResample,
 * 23 DfqJpegImage, 24 DfqJpegSegment, 25 DfqJpegDecode, 26 DfqJpegHuff, 27 DfqJpegTables, 28 DfqAbsorb,
 * 29 DfqPngImage, 30 DfqPngDecode; 20 is
 * unassigned and returns -1, as ABI 11 released it): lets a binding verify
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
                         DFQ_LAYER_FOLD_PENDING, DFQ_LAYER_ROWS_READY: see below                */
  int64_t cmin_off;   /* [2][C of rel_in] running column minima, double-buffered by sweep parity
                         (scratch, valid when rel_in >= 0)                                  */
  int64_t cmax_off;   /* [2][C of rel_in] running column maxima                              */
  int64_t fold_off;   /* DFQ_LAYER_FOLD_PENDING: [rows] fold factors gamma/sqrt(var+eps) (DfqFold.fac_off)      */
  int64_t rext_off;   /* DFQ_LAYER_ROWS_READY: [2][rows] scratch, row minima then row maxima (DfqFold.scan_rows)     */
  int32_t rext_rows;  /* DFQ_LAYER_ROWS_READY: 0 = the extrema of every row are in rext_off; n > 0 = only those of rows
                         [0, min(n, rows)) are (DfqFold.row_prefix): dfq_cle_run completes the rest                   */
  int32_t _pad;
} DfqLayer;

/* The flags are promises about the call that runs RIGHT AFTER dfq_bn_fold, on the same weights:
 *   DFQ_LAYER_COLS_READY   the fold (scan_go > 0) has written buffer 0 of the column extrema of the FOLDED weights.
 *   DFQ_LAYER_FOLD_PENDING the fold ran with DfqFold.mode = DFQ_FOLD_DEFER: biases, BN vectors and the factors at fold_off
 *                          are final, the weights are NOT yet multiplied by the factors.  dfq_cle_run completes the fold:
 *                          k_cle_stack multiplies each row by its factor as its first sweep reads it (fl(w * f), the value
 *                          the fold would have stored); on every other path (the engine, no sweep at all) the fold is
 *                          applied to the weights before anything else.  Either way the weights are folded on return.
 *   DFQ_LAYER_ROWS_READY   the fold (DfqFold.scan_rows) has written the row extrema of the FOLDED weights of this `first`
 *                          layer to rext_off.  When every first layer of a k_cle_stack run carries it, the kernel may
 *                          derive the scales of the first two sweeps from these extrema and the column extrema alone and
 *                          apply both sweeps in one pass over the weights (DfqCleResult.fused_sweeps); the scratch is
 *                          consumed either way (its content after the call is unspecified).
 *                          With rext_rows > 0 only a prefix of the rows was scanned.  The kernel's guard then decides from
 *                          that prefix where it can (every metric term is >= 0, so a partial sum is a lower bound too) and
 *                          derives the other rows' extrema while the fused pass holds them; where it cannot, it scans the
 *                          remaining rows itself first and decides as with a full scan (DfqCleResult.rows_streamed). */
#define DFQ_LAYER_COLS_READY 1
#define DFQ_LAYER_FOLD_PENDING 2
#define DFQ_LAYER_ROWS_READY 4

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
  int32_t fused_sweeps;    /* 2: k_cle_stack applied sweeps 1 and 2 in one pass (DFQ_LAYER_ROWS_READY), 0: one pass
                              per sweep.  Results are the same bits either way.                                  */
  int32_t bc_prepared;     /* 1: the attached bias correction (dfq_cle_run's bc tables) holds the results of the final
                              weights - the fused pass ran and every group stopped after sweep 2.  0: none attached, or
                              its scratch is stale (all or nothing).                                              */
  int32_t rows_streamed;   /* first layers that arrived with a row prefix (DfqLayer.rext_rows): DFQ_ROWS_* below     */
  int32_t _pad;
} DfqCleResult;
/* DfqCleResult.rows_streamed:
 *   DFQ_ROWS_FULL       no first layer arrived with a prefix (or none was shorter than its rows)
 *   DFQ_ROWS_STREAMED   the prefix decided the guard for every group; the fused pass derived the other rows' extrema
 *   DFQ_ROWS_UNDECIDED  the prefix left some group undecided: the remaining rows were scanned, then the full guard ran
 *   DFQ_ROWS_HOST_FULL  the prefix could not be used (no fused pass possible, or s_range with lo <= 0 or hi = inf):
 *                       the remaining rows were scanned, then the full guard ran (where a fused pass is possible) */
#define DFQ_ROWS_FULL 0
#define DFQ_ROWS_STREAMED 1
#define DFQ_ROWS_UNDECIDED 2
#define DFQ_ROWS_HOST_FULL 3

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

/* dfq_cle_run with an attached bias correction (bc, n_bc, bc_terms, n_bc_terms, bc_num_bits; NULL or 0: none, which is
 * dfq_cle_run).  One level of a dfq_bias_correct table (same structs, same meaning, num_bits = bc_num_bits) whose
 * correction k_cle_stack computes inside its fused pass, from the rows it holds in shared memory - instead of a later pass
 * that reads the corrected layers again.  The call writes each entry's minmax_off, expect_off and delta_off (eps . E[x])
 * and nothing else: no bias and no fake_bias changes.  Those are the results of the final weights only when
 * result->bc_prepared is 1; a dfq_bias_correct of the same table with every entry flagged DFQ_BC_PREPARED then only
 * retires them.  Refused (DFQ_E_ARG) unless the problem runs on k_cle_stack and every entry is the `second` layer of a
 * relation, listed once, with flags 0 and expect_len = cols. */
struct DfqBcLayer;
struct DfqExpectTerm;
int dfq_cle_run_bc(float* arena, int64_t arena_floats,
                   const DfqLayer* layers, int32_t n_layers,
                   const DfqRelation* rels, int32_t n_rels,
                   const int32_t* step_ptr, const int32_t* step_layers, int32_t n_steps,
                   const DfqCleParams* params, DfqCleResult* result,
                   int32_t n_groups, int32_t* group_sweeps,
                   const struct DfqBcLayer* bc, int32_t n_bc, const struct DfqExpectTerm* bc_terms, int32_t n_bc_terms,
                   int32_t bc_num_bits, void* stream);

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
  int32_t scan_rows;          /* _DEFER only, 1: also write the row extrema of the FOLDED weights to the layer's rext_off
                                 ([0, rows) minima, [rows, 2 rows) maxima; layers[] must carry it).  0: no row scan.    */
  int64_t fac_off;            /* _DEFER, _APPLY: [rows] fold factors gamma/sqrt(var+eps)                              */
  int32_t row_prefix;         /* with scan_rows: 0 = scan every row, n > 0 = only rows [0, min(n, rows)) (DfqLayer.rext_rows;
                                 the layer must not also be column-scanned).  Ignored without scan_rows.             */
  int32_t _pad;
} DfqFold;
/* DFQ_FOLD_FULL   the fold above: weights, bias, fake_weight / fake_bias.
 * DFQ_FOLD_DEFER  everything but the weights: bias, fake_weight / fake_bias, and each row's factor into fac_off.  With
 *                 scan_go > 0 the weights are READ (not written) and the column extrema of fl(w * factor) - those of the
 *                 folded weights - go to buffer 0; with scan_rows the row extrema of fl(w * factor) go to rext_off.  The weights stay unfolded until a DFQ_LAYER_FOLD_PENDING layer entry
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
                                subtracting it (dfq.py:292); DFQ_BC_PREPARED: see below */
  int64_t expect_off;        /* scratch [expect_len] */
  int64_t delta_off;         /* scratch/out [rows]: eps . E[x]                           */
  int64_t next_bn_b_off;     /* fake_bias that receives -delta (dfq.py:204-206), or -1  */
  int64_t minmax_off;        /* scratch [2]: per-tensor min/max of W                     */
  int64_t colmin_off;        /* n_col > 0: [n_col] column minima / maxima of the CURRENT weights that the caller vouches */
  int64_t colmax_off;        /* for; the per-tensor range (dfq.py:14) is reduced from them and the weights are not      */
  int32_t n_col;             /* streamed a second time.  After dfq_cle_run the valid buffer of a `second` layer is      */
  int32_t _pad;              /* cmin_off + (group_sweeps[group] & 1) * C (same for cmax).  0: scan the weights.          */
} DfqBcLayer;
/* DFQ_BC_PREPARED: delta_off, expect_off and minmax_off already hold this layer's results for its CURRENT weights (a
 * dfq_cle_run with this table attached reported bc_prepared, and nothing has touched the arena since).  When every entry
 * carries it, dfq_bias_correct only retires the deltas: bias = fl(bias - delta), next fake_bias = fl(fake_bias - delta),
 * no weight is read.  A table that mixes flagged and unflagged entries, or flags a raw-sum entry, is refused. */
#define DFQ_BC_PREPARED 4
int dfq_bias_correct(float* arena, int64_t arena_floats, const DfqLayer* layers, int32_t n_layers,
                     const DfqBcLayer* bc, int32_t n_bc, const DfqExpectTerm* terms, int32_t n_terms,
                     const int32_t* level_ptr, int32_t n_levels, int32_t num_bits, void* stream);

/* Bias absorption and weight clipping inside the bias correction: what the separate calls
 *   bias_absorption(graph, relations, bottoms, N)   dfq.py:121-164
 *   clip_weight(graph, [lo, hi], targ)              dfq.py:167-170
 *   bias_correction(graph, bottoms, targ)           dfq.py:173-293
 * compute one after the other, with each corrected weight row read once.  One DfqAbsorb per absorbing relation (the
 * caller decides which relations absorb: a torch.nn.ReLU between the layers, dfq.py:123-130): */
typedef struct DfqAbsorb {
  int32_t first, second;     /* layer indices of the relation */
  int32_t n;                 /* channels = first.rows = groups * second.cols */
  int32_t _pad;
  int64_t bn_w_off, bn_b_off;  /* the relation's BN fake_weight / fake_bias (after equalization) */
  int64_t c_off;             /* scratch/out [n]: c = clamp(fake_bias - N * fake_weight, 0) (dfq.py:143-144) */
} DfqAbsorb;
/* Before the correction: c of every relation, fake_bias -= c, and first.bias -= c when `first` has no correction entry.
 * The `second` layer of every relation needs an entry: a raw-sum entry (flags bit 0, its terms holding c) is the
 * absorption alone; any other entry adds (sum_k W) . c of the UNCLIPPED row to the bias, per group as dfq.py:150-153.
 * clip != 0: every weight of `layers` is clamped to [clip_lo, clip_hi] in the arena - those of the entries while their rows
 * are read (the correction's quantization error and per-tensor range are those of the clamped weights), the others in one
 * more launch.  Biases are never clipped.  The bias of an entry rounds as the separate calls do:
 * fl(fl(fl(b + wc) - c) - delta).  n_bc = 0: the clip alone.
 * Refused: a non-finite absorb_n, a clip range that is not finite with lo <= hi, DFQ_BC_PREPARED entries. */
int dfq_bias_correct_absorb_clip(float* arena, int64_t arena_floats, const DfqLayer* layers, int32_t n_layers,
                                 const DfqBcLayer* bc, int32_t n_bc, const DfqExpectTerm* terms, int32_t n_terms,
                                 const int32_t* level_ptr, int32_t n_levels, int32_t num_bits,
                                 const DfqAbsorb* absorb, int32_t n_absorb, float absorb_n,
                                 int32_t clip, float clip_lo, float clip_hi, void* stream);

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

/* The convolution's fp32 output in pixel-major rows, for detection heads whose outputs are permuted to [N, OH, OW, O] and
 * concatenated along the anchors (`permute(0, 2, 3, 1).contiguous().view(N, -1, k)` then `torch.cat(..., 1)`):
 *   v = clamp(clamp(fp32(fp32_rn(acc) * dq[o]) + bias[o], pre), post)      as dfq_i8_conv_fused computes it
 *   e->y[n * img_stride + off + p * O + o] = v                             p = oh * OW + ow
 * Each image's OH * OW * O floats start at `off` inside its img_stride floats, so rows [off / k, off / k + OH * OW * O / k) of
 * an [N, R, k] tensor (img_stride = R * k) are this layer's slice of the concatenation; nothing else of y is written.  Only
 * e->y and the two clamps of *e are used.  DFQ_E_ARG, with a reason: y NULL or not 4-byte aligned, residual or yq not NULL,
 * off < 0, img_stride < off + OH * OW * O, NaN or unordered bounds in either clamp, y's extent overlapping xq.  Grouping
 * as dfq_i8_conv. */
int dfq_i8_conv_nhwc(const int8_t* xq, const int8_t* wq, const float* dq, const float* bias, const DfqI8Epilogue* e,
                     int64_t off, int64_t img_stride, const DfqI8Conv* g, void* stream);

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

/* Bilinear resize to a given size (F.interpolate(x, size=(OH, OW), mode='bilinear', align_corners=...)). */
typedef struct DfqI8Resize {
  int32_t N, C, H, W;          /* fp32 NCHW input                                                                 */
  int32_t OH, OW;              /* output size (the `size=` of F.interpolate)                                      */
  int32_t align_corners;       /* 0 or 1                                                                          */
  int32_t coff, cstride;       /* codes go to channels [coff, coff + round_up(C, 16)) of int8 NHWC [N, OH, OW, cstride] */
  float out_scale, lo, hi;     /* q(clamp(v, lo, hi), out_scale); (-inf, +inf): no clamp                          */
} DfqI8Resize;
/* x fp32 NCHW [N, C, H, W] -> y fp32 NCHW [N, C, OH, OW] (NULL: not written), bit for bit torch's CUDA upsample_bilinear2d
 * of a contiguous NCHW fp32 tensor with no scale_factor: per axis scale = align_corners ? (in - 1) / (out - 1) (0 when
 * out == 1) : in / out in fp32, source index scale * dst or max(scale * (dst + 0.5) - 0.5, 0) with torch's fused
 * multiply-adds, and a plain copy when the size does not change; and / or yq[m * cstride + coff + c] =
 * q(clamp(y, lo, hi), out_scale) (NULL: not written), the clamp keeping NaN.  The codes are those of the fp32 value, so
 * NaN, +-inf, -0.0 and subnormal inputs give what the per-layer path gives.  Pad channels C .. round_up(C, 16) of the slice
 * are written 0 and nothing outside the slice.  DFQ_E_ARG, with a reason: a non-positive size, align_corners not 0 / 1,
 * coff or cstride not a multiple of 16 or the slice not inside cstride, no output, yq not 16-byte aligned or x / y not
 * 4-byte aligned, an out_scale that is not finite and non-negative while yq is written, NaN or unordered bounds, x
 * overlapping y or the slice, y overlapping the slice. */
int dfq_i8_upsample_bilinear(const float* x, float* y, int8_t* yq, const DfqI8Resize* g, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Int8 execution under the reference's own quantization: asymmetric per-tensor min / max, b <= 8 bits
 *
 * The state main_cls.py:196 runs: quantize_targ_layer has written w^ = fp32(fp32(qw * fw) + mw) into the weights (one
 * (fw, mw) per tensor, codes qw in [0, 2^b - 1]) and QuantMeasure turns the input into x^ = fp32(fp32(qa * fa) + ma) with
 *   ma = running_min,  s_a = max((running_max - running_min) / (2^b - 1), 1e-8) in double,  fa = fp32(s_a),
 *   qa = rint(clamp(fp32(fp32(x + (-ma)) * fp32(1 / s_a)), 0, 2^b - 1))     (CUDA: the division is a reciprocal multiply)
 * Codes are stored shifted, q' = q - 128, in the layouts of dfq_i8_quantize_nhwc / dfq_i8_pack_weights, and the shift goes
 * into the offsets ma' = ma + 128 fa, mw' = mw + 128 fw.  Per output element, over the in-image taps only (padding is a
 * dequantized 0.0 in the fake-quantized model, not a code):
 *   y = fp32(kP P + kA A + kW Wv + kN Nv) + bias[o]      each product and sum a double op, in this order, no FMA
 *   P = sum qa' qw' (int32),  A = sum qa',  Wv = sum qw',  Nv = (in-image taps) * C / groups
 *   kP = fa fw,  kA = fa mw',  kW = ma' fw,  kN = ma' mw'  (formed in double by the caller)
 * This is the value of sum (qa fa + ma)(qw fw + mw) rounded to fp32 once; the fake-quantized model sums the rounded
 * products x^ w^ in fp32, so the two agree to fp32 rounding, not bit for bit.  Grouping as dfq_i8_conv.  K = kh * kw * C /
 * groups must stay below 131072 (codes of -128 reach the main loop and K * 128 * 128 must stay below 2^31): DFQ_E_UNSUPPORTED,
 * as are codes of more than 8 bits.
 * ------------------------------------------------------------------------------------------- */
typedef struct DfqI8Affine {
  double kP, kA, kW, kN;
} DfqI8Affine;
/* fp32 NCHW x -> int8 NHWC q[N, H, W, Cpad] = qa - 128 (pad channels 0) and int32 S[N, H, W] = sum of q over the C real
 * channels, with QuantMeasure's scalars of the range (act_min, act_max) at num_bits: fp32((q + 128) * fa) + ma is
 * QuantMeasure's output bit for bit, +-inf included.  NaN has no code there (its output is NaN); here it gets qa = 0.
 * q 16-byte aligned.  DFQ_E_ARG: a non-finite range or scale, num_bits < 1; DFQ_E_UNSUPPORTED: num_bits > 8. */
int dfq_i8_affine_quantize(const float* x, int8_t* q, int32_t* S, int32_t N, int32_t C, int32_t H, int32_t W, int32_t Cpad,
                           float act_min, float act_max, int32_t num_bits, void* stream);
/* Weight codes of a fake-quantized tensor w^ (layout as dfq_i8_pack_weights): qw = clamp(rint(fp32(fp32(w^ - w_min) /
 * w_scale)), 0, 2^b - 1), stored qw - 128; *n_bad (device int32, zeroed by the call) = the weights with
 * fp32(fp32(qw * w_scale) + w_min) != w^ bit for bit.  Dense layers also get table[O][(kh + 1) * (kw + 1)], the prefix
 * sums of their codes over the taps (T[r][s] = sum over taps r' < r, s' < s and all channels); depthwise layers take
 * table = NULL.  DFQ_E_ARG: non-finite w_min, w_scale not finite and positive; refusals as dfq_i8_affine_conv. */
int dfq_i8_affine_pack(const float* w, float w_min, float w_scale, int32_t num_bits, int8_t* packed, int32_t* table,
                       int32_t* n_bad, const DfqI8Conv* g, void* stream);
/* The convolution with the epilogue above: xq and S from dfq_i8_affine_quantize (S unused by depthwise layers), wq and
 * table from dfq_i8_affine_pack, bias[O] (NULL: none), y fp32 NCHW [N, O, OH, OW]; acc_out (NULL: not written) receives P.
 * DFQ_E_ARG: non-finite constants, a dense layer without S or table; DFQ_E_UNSUPPORTED: K >= 131072, other groupings. */
int dfq_i8_affine_conv(const int8_t* xq, const int32_t* S, const int8_t* wq, const int32_t* table, const DfqI8Affine* k,
                       const float* bias, float* y, int32_t* acc_out, const DfqI8Conv* g, void* stream);
/* The affine residual epilogue of dfq_i8_affine_conv_fused, for layers chained through the next layer's codes.  Per output
 * element (n, o, p), the ops of the per-layer path in its order:
 *   v  = fp32(kP P + kA A + kW Wv + kN Nv) + bias[o]          as dfq_i8_affine_conv
 *   v  = v < pre_lo ? pre_lo : (v > pre_hi ? pre_hi : v)       NaN stays NaN
 *   v  = fp32(v + residual[n, o, p])                           only when residual != NULL: fp32 NCHW [N, O, OH, OW]
 *   v  = v < post_lo ? post_lo : (v > post_hi ? post_hi : v)
 *   y[n, o, p]  = v                                            when y != NULL: fp32 NCHW [N, O, OH, OW]
 *   yq[n, p, o] = the code dfq_i8_affine_quantize gives v at (out_min, out_max, out_bits), the CONSUMER's range: int8 NHWC
 *                 [N, OH, OW, round_up(O, 16)] when yq != NULL, pad channels 0 (NaN -> -128, +-inf saturate)
 *   S[n, p]     = the sum of yq[n, p, :] over the O real channels (int32 [N, OH, OW]) when S != NULL: what
 *                 dfq_i8_affine_quantize writes, bit for bit, for a dense consumer
 * No clamp is (-inf, +inf). */
typedef struct DfqI8AffineEpilogue {
  const float* residual;
  float* y;
  int8_t* yq;
  int32_t* S;
  float out_min, out_max;
  int32_t out_bits;
  float pre_lo, pre_hi, post_lo, post_hi;
} DfqI8AffineEpilogue;
/* The convolution of dfq_i8_affine_conv (inputs as there: xq and S_in, the layer's own input codes and sums) with the
 * epilogue *e.  When S is written by more than one tile (O > 64 dense, O > 16 depthwise) the call zeroes it on `stream`
 * first and the kernel adds into it.  DFQ_E_ARG, with a reason: y and yq both NULL, S without yq, yq not 16-byte aligned,
 * residual, y or S not 4-byte aligned, NaN or unordered bounds in either clamp, and while yq is written an output range
 * dfq_i8_affine_quantize refuses (non-finite, or a scale that is not a finite fp32 number) or out_bits < 1; outputs that
 * overlap each other or the residual (extents from the geometry).  DFQ_E_UNSUPPORTED: out_bits > 8.  Refusals of
 * dfq_i8_affine_conv as there. */
int dfq_i8_affine_conv_fused(const int8_t* xq, const int32_t* S_in, const int8_t* wq, const int32_t* table,
                             const DfqI8Affine* k, const float* bias, const DfqI8AffineEpilogue* e, const DfqI8Conv* g,
                             void* stream);
/* The observers the reference's replace_op() puts on functional ops (QuantMeasure in eval mode without update_stat), run in
 * the affine epilogue.  With fq(t, lo, hi, b) = what QuantMeasure returns for t at running_min lo, running_max hi and
 * num_bits b on a CUDA tensor (the double prologue of the fake quantization, a reciprocal multiply, rint, clamp to
 * [0, 2^b - 1], fp32(fp32(q * scale) + min); NaN stays NaN, +-inf saturate), dfq_i8_affine_conv_observed computes per
 * output element, in this order:
 *   v  = fp32(kP P + kA A + kW Wv + kN Nv) + bias[o]          as dfq_i8_affine_conv
 *   v  = v < pre_lo ? pre_lo : (v > pre_hi ? pre_hi : v)
 *   v  = fq(v, obs_min, obs_max, obs_bits)                     when obs_bits > 0: the observer on the fused operand
 *   r  = fq(residual[n, o, p], res_min, res_max, res_bits)     when res_bits > 0 (residual[n, o, p] when 0)
 *   v  = fp32(v + r)                                           only when residual != NULL
 *   v  = v < post_lo ? post_lo : (v > post_hi ? post_hi : v)
 *   y, yq and S as dfq_i8_affine_conv_fused.
 * An observer with bits 0 is off. */
typedef struct DfqI8AffineObserve {
  float obs_min, obs_max;
  int32_t obs_bits;
  float res_min, res_max;
  int32_t res_bits;
} DfqI8AffineObserve;
/* dfq_i8_affine_conv_fused with the observers *o.  Refusals of dfq_i8_affine_conv_fused as there, and DFQ_E_ARG with a
 * reason: o NULL, an observer with bits < 0 or (when on) a non-finite range or a scale that is not a finite fp32 number,
 * res_bits > 0 without a residual, both observers off (dfq_i8_affine_conv_fused computes that).  DFQ_E_UNSUPPORTED: an
 * observer with bits > 8.  Nothing is written when a call is refused. */
int dfq_i8_affine_conv_observed(const int8_t* xq, const int32_t* S_in, const int8_t* wq, const int32_t* table,
                                const DfqI8Affine* k, const float* bias, const DfqI8AffineEpilogue* e,
                                const DfqI8AffineObserve* o, const DfqI8Conv* g, void* stream);
/* Where dfq_i8_affine_conv_layout puts its codes and S, and what its out-of-image taps read. */
typedef struct DfqI8AffineLayout {
  int32_t coff, cstride;       /* codes go to channels [coff, coff + round_up(O, 16)) of int8 NHWC [N, OH, OW, cstride]    */
  int32_t S_accumulate;        /* 1: add the pixels' sums into S, which the caller zeroed (a concatenation's writers)       */
  int32_t pad_code_on;         /* 1: every out-of-image tap reads the shifted code pad_code over the C real channels        */
  int32_t pad_code;            /* in [-128, 127]                                                                           */
} DfqI8AffineLayout;
/* dfq_i8_affine_conv_observed (o != NULL) or dfq_i8_affine_conv_fused (o == NULL) with the layout *l:
 *   yq[n, p, coff + o] = the code of v (pad channels O .. round_up(O, 16) written 0, nothing else of the row), pixel p's
 *                 codes cstride bytes after pixel p - 1's: the producers of a channel concatenation write the consumer's
 *                 input directly;
 *   S[n, p]     += the sum of the slice's codes over its O real channels when S_accumulate (S zeroed by the caller once
 *                 for all the concatenation's writers), else as dfq_i8_affine_conv_fused;
 *   pad_code_on: y, yq and S equal, bit for bit, those of the same call with padding 0 on the input padded by pad_h rows
 *                 and pad_w columns on each side whose padded pixels hold the code pad_code in every real channel (what
 *                 the per-layer path computes on F.pad(x): its zeros become the code of +0.0 at the layer's input range).
 *                 Dense layers correct P, A, Wv and Nv from the prefix table; depthwise layers read the code in the loop.
 * Refusals of dfq_i8_affine_conv_observed / _fused as there (overlaps taken over the slice's extent), and DFQ_E_ARG with a
 * reason: l NULL, coff or cstride not a multiple of 16, the slice past cstride, S_accumulate or pad_code_on not 0 / 1, a
 * pad code outside [-128, 127].  Nothing is written when a call is refused. */
int dfq_i8_affine_conv_layout(const int8_t* xq, const int32_t* S_in, const int8_t* wq, const int32_t* table,
                              const DfqI8Affine* k, const float* bias, const DfqI8AffineEpilogue* e,
                              const DfqI8AffineObserve* o, const DfqI8AffineLayout* l, const DfqI8Conv* g, void* stream);
/* Bilinear resize into a concatenation's codes under the affine scheme. */
typedef struct DfqI8AffineResize {
  int32_t N, C, H, W, OH, OW, align_corners, coff, cstride;   /* as DfqI8Resize                                      */
  float pre_lo, pre_hi;                                        /* clamp before the observer                           */
  float obs_min, obs_max;                                      /* the observer on the concatenation operand           */
  int32_t obs_bits;                                            /* 0: off                                              */
  float post_lo, post_hi;                                      /* clamp after it                                      */
  float out_min, out_max;                                      /* the consumer's range                                */
  int32_t out_bits;
} DfqI8AffineResize;
/* x fp32 NCHW [N, C, H, W] -> per output value, in this order: v = dfq_i8_upsample_bilinear's y (torch's
 * upsample_bilinear2d bit for bit), clamp(v, pre), fq(v, obs) when obs_bits > 0 (as dfq_i8_affine_conv_observed),
 * clamp(v, post), then yq[n, p, coff + c] = the code dfq_i8_affine_quantize gives v at (out_min, out_max, out_bits), pad
 * channels 0, nothing outside the slice; S[n, p] += the slice's sum over its C real channels (S NULL: not written; the
 * caller zeroes S).  DFQ_E_ARG, with a reason: a non-positive size, align_corners not 0 / 1, coff or cstride not a multiple
 * of 16 or the slice past cstride, x or yq NULL, yq not 16-byte aligned or x / S not 4-byte aligned, NaN or unordered
 * bounds, an observer or output range as dfq_i8_affine_conv_observed refuses, x, the slice and S overlapping.
 * DFQ_E_UNSUPPORTED: obs_bits or out_bits above 8.  Nothing is written when a call is refused. */
int dfq_i8_affine_upsample_bilinear(const float* x, int8_t* yq, int32_t* S, const DfqI8AffineResize* g, void* stream);
/* A detection head's rows under the affine scheme (dfq_i8_conv_nhwc's layout): the convolution of dfq_i8_affine_conv
 * (inputs as there) with, per output element (n, o, p), in this order:
 *   v = fp32(kP P + kA A + kW Wv + kN Nv) + bias[o]           as dfq_i8_affine_conv
 *   v = clamp(v, pre_lo, pre_hi)                               NaN stays NaN; (-inf, +inf): no clamp
 *   v = fq(v, obs_min, obs_max, obs_bits)                      when obs_bits > 0: the concatenation operand's observer
 *   v = clamp(v, post_lo, post_hi)
 *   v = fq(v, tail_min, tail_max, tail_bits)                   when tail_bits > 0: the observer of the concatenation's
 *                                                              single user (elementwise, so per slice)
 *   y[n * img_stride + off + p * O + o] = v
 * fq as dfq_i8_affine_conv_observed.  Nothing else of y is written. */
typedef struct DfqI8AffineRows {
  float* y;
  int64_t off, img_stride;     /* the slice of each image's img_stride floats; img_stride >= off + OH * OW * O      */
  float pre_lo, pre_hi, post_lo, post_hi;
  float obs_min, obs_max;
  int32_t obs_bits;            /* 0: off                                                                          */
  float tail_min, tail_max;
  int32_t tail_bits;           /* 0: off                                                                          */
} DfqI8AffineRows;
/* Refusals of dfq_i8_affine_conv as there, and DFQ_E_ARG with a reason: r or y NULL, y not 4-byte aligned, NaN or
 * unordered bounds, off < 0, img_stride < off + OH * OW * O, the rows overlapping xq or S_in, an observer with bits < 0
 * or (when on) a non-finite range or a scale that is not a finite fp32 number.  DFQ_E_UNSUPPORTED: an observer with bits
 * > 8.  Nothing is written when a call is refused. */
int dfq_i8_affine_conv_rows(const int8_t* xq, const int32_t* S_in, const int8_t* wq, const int32_t* table,
                            const DfqI8Affine* k, const float* bias, const DfqI8AffineRows* r, const DfqI8Conv* g,
                            void* stream);
/* dfq_i8_maxpool under the affine scheme; the geometry and the two modes as there (exactly one input):
 *   xq (codes): shifted codes int8 NHWC [N, H, W, Cpad] -> yq, the byte-wise signed max of the taps inside the input.  The
 *      shifted code of dfq_i8_affine_quantize is monotone non-decreasing (its scale is at least 1e-8), so this is the code
 *      of max_pool2d(v) for any window without NaN.  A window with no tap in the input gives -128, the code of torch's
 *      -inf; pad channels 0.  The exception of the per-layer path: a window holding a NaN gives -128 there (NaN quantizes
 *      to code 0) and the max of the other codes here.  y must be NULL; out_min, out_max and out_bits are not read.
 *   x (fp32): NCHW -> y (NULL: not written) bit for bit torch's CUDA max_pool2d, as dfq_i8_maxpool, and / or yq = the codes
 *      dfq_i8_affine_quantize gives y at (out_min, out_max, out_bits), the consumer's range (NULL: not written).
 * Both: S[n, p] = the sum of yq[n, p, :] over the C real channels (int32 [N, OH, OW]; NULL: not written), what
 * dfq_i8_affine_quantize writes bit for bit; the call zeroes it on `stream` and the kernel adds into it.
 * Refusals of dfq_i8_maxpool as there, and DFQ_E_ARG with a reason: S without yq or not 4-byte aligned, inputs and outputs
 * S included overlapping, and while yq is written in fp32 mode an output range dfq_i8_affine_quantize refuses or
 * out_bits < 1.  DFQ_E_UNSUPPORTED: out_bits > 8 in that case.  Nothing is written when a call is refused. */
int dfq_i8_affine_maxpool(const int8_t* xq, const float* x, float* y, int8_t* yq, int32_t* S, float out_min, float out_max,
                          int32_t out_bits, const DfqI8Pool* g, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ncnn int8 model files (dfq_b200/ncnn.py): the weight codes as the file holds them, and ncnn's mean of a plane
 * ------------------------------------------------------------------------------------------- */
/* int8 codes in ncnn's weight layout [O][C/groups][kh][kw] -> the packed layout of dfq_i8_pack_weights (groups == 1:
 * [O][kh][kw][Cpad]; depthwise: [kh*kw][Cpad]; pad channels 0), copied verbatim: no scale, no rounding.  Uses g's O, C,
 * kh, kw, groups and Cpad; refusals of dfq_i8_pack_weights, and DFQ_E_ARG with a reason: a NULL pointer, codes and packed
 * overlapping. */
int dfq_i8_pack_codes(const int8_t* codes, int8_t* packed, const DfqI8Conv* g, void* stream);
/* The inverse: the codes [O][C/groups][kh][kw] of a packed layer (pad channels are not read).  Refusals as
 * dfq_i8_pack_codes. */
int dfq_i8_unpack_codes(const int8_t* packed, int8_t* codes, const DfqI8Conv* g, void* stream);
/* ncnn's mean of each (image, channel) plane of x fp32 [N, C, P] (contiguous), in ncnn's order:
 *   sum = 0.f;  for p in 0 .. P - 1: sum = fp32(sum + x[n, c, p])         sequential, every add rounded
 *   v   = divide ? fp32(sum / P) : fp32(sum * fp32(1 / P))                   Pooling global average : Reduction MEAN
 * (a reading of ncnn's pooling.cpp and reduction.cpp, coeff 1).  y fp32 [N, C] receives v (NULL: not written), and / or
 * yq int8 [N, round_up(C, 16)] the consumer's codes q8(v, out_scale) as dfq_i8_quantize_nhwc forms them (roundf, clamp
 * +-127, NaN -> -127), pad channels 0 (NULL: not written) - the codes a chained 1 x 1 layer reads as [N, 1, 1, Cpad].
 * No host synchronisation.  DFQ_E_ARG with a reason: x NULL, y and yq both NULL, N, C or P not positive, divide not 0 or
 * 1, x or y not 4-byte aligned, yq not 16-byte aligned, out_scale not finite and non-negative while yq is written, x
 * past 2^63 bytes, x, y and yq overlapping. */
int dfq_i8_plane_mean(const float* x, float* y, int8_t* yq, int64_t N, int32_t C, int64_t P, int32_t divide, float out_scale,
                      void* stream);

/* ---------------------------------------------------------------------------------------------
 * SSD post-processing (modeling/detection/predictor.py Predictor.predict, utils/detection/box_utils.py) for a batch
 * ------------------------------------------------------------------------------------------- */
typedef struct DfqSsdNms {
  int32_t N, P, C;               /* images, priors, classes (class 0 is the background)                               */
  int32_t prior_batch;           /* priors [prior_batch, P, 4]: 1 (shared by every image) or N                        */
  float center_variance, size_variance;
  float prob_threshold;          /* candidates: score > prob_threshold (strict: NaN never is one)                     */
  float iou_threshold;           /* a remaining box is kept while iou_of(box, picked) <= iou_threshold                */
  int32_t candidate_size;        /* the best candidate_size candidates of a class enter NMS, 1 .. 1024                */
  int32_t top_k;                 /* > 0: at most top_k picks per class; <= 0: no limit                                */
} DfqSsdNms;
/* convert_locations_to_boxes + center_form_to_corner_form, bit for bit torch's CUDA ops: per (image n, prior p), with
 * l = locations[n, p], q = priors[prior_batch == 1 ? 0 : n, p] (centre form), every op rounded to fp32 in this order:
 *   cx = (l0 * cv) * q2 + q0,  cy = (l1 * cv) * q3 + q1,  w = expf(l2 * sv) * q2,  h = expf(l3 * sv) * q3
 *   boxes[n, p] = (cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2)
 * locations and boxes fp32 [N, P, 4].  Reads N, P, prior_batch and the variances of *d.  DFQ_E_ARG, with a reason: d
 * NULL, N or P < 1, prior_batch neither 1 nor N, a NULL or not 16-byte aligned pointer. */
int dfq_ssd_decode(const float* locations, const float* priors, float* boxes, const DfqSsdNms* d, void* stream);
/* Per (image n, class c = 1 .. C-1) of scores fp32 [N, P, C] and the decoded boxes fp32 [N, P, 4]: the candidates
 * (score > prob_threshold) ordered by score descending, -0.0 equal to +0.0, ties broken by the lower prior index (the
 * reference's CPU sort is not stable; this is the one place the result may differ from it); the first candidate_size of
 * them; then box_utils.hard_nms: pick the first remaining, stop once top_k > 0 picks are made, drop every remaining box r
 * with !(iou_of(r, picked) <= iou_threshold), iou_of in the reference's fp32 op order with NaN-propagating max, min and
 * clamp.  Writes, for segment s = n * (C - 1) + c - 1, its picks in pick order to slot_boxes fp32 [N * (C - 1),
 * candidate_size, 4] and slot_probs [N * (C - 1), candidate_size] (the candidates' scores), their number to counts[s]
 * (int32 [N * (C - 1)]), and the exclusive scan of counts to offsets (int64 [N * (C - 1) + 1]; offsets[n * (C - 1)] is
 * where image n starts in the flat output, the last entry the total).  DFQ_E_ARG, with a reason: the refusals of
 * dfq_ssd_decode, C < 2, candidate_size < 1, boxes or slot_boxes not 16-byte aligned.  DFQ_E_UNSUPPORTED: candidate_size
 * above 1024, N * (C - 1) above INT32_MAX. */
int dfq_ssd_nms(const float* scores, const float* boxes, float* slot_boxes, float* slot_probs, int32_t* counts,
                int64_t* offsets, const DfqSsdNms* d, void* stream);
/* The flat output of the picks dfq_ssd_nms left in the slots, what Predictor.predict returns for each image in turn:
 * out_boxes fp32 [T, 4] (times (w, h, w, h) of image_sizes fp32 [N, 2] = (width, height) per image, unscaled when
 * image_sizes is NULL), out_labels int64 [T] = c, out_probs fp32 [T]; T = offsets[N * (C - 1)].  Classes ascending, picks
 * in pick order.  Refusals of dfq_ssd_nms, and DFQ_E_ARG for a NULL output or out_boxes not 16-byte aligned. */
int dfq_ssd_compact(const float* slot_boxes, const float* slot_probs, const int32_t* counts, const int64_t* offsets,
                    const float* image_sizes, float* out_boxes, int64_t* out_labels, float* out_probs, const DfqSsdNms* d,
                    void* stream);
/* box_utils.soft_nms per (image n, class c = 1 .. C-1), as Predictor.predict calls it with nms_method "soft": of scores
 * fp32 [N, P, C] and the decoded boxes fp32 [N, P, 4], the candidates (score > prob_threshold) in prior order; then, until
 * no row remains: pick the first row of the largest score (NaN the largest), emit its box and current score, stop once
 * top_k > 0 picks are made or it was the only row, move the last row into its place and drop the last row, rescore every
 * row s = fl(s * expf(fl(fl(-fl(iou * iou)) / sigma))) with iou = iou_of(picked, row) in the reference's op order, and
 * keep the rows with s > prob_threshold in order.  expf is CUDA's precise expf (torch's exp on a CUDA tensor); every
 * other op is the reference's, bit for bit.  candidate_size and iou_threshold are not read.
 * Writes the candidate count of segment s = n * (C - 1) + c - 1 to candidates[s] and its pick count to counts[s] (both
 * int32 [N * (C - 1)]), and the exclusive scan of counts to offsets (int64 [N * (C - 1) + 1], as dfq_ssd_nms).  Segments
 * of more than 11,264 candidates hold their rows in global memory: the call then allocates 20 * P bytes per SM on
 * `stream` and frees them there.  DFQ_E_ARG, with a reason: the refusals of dfq_ssd_decode, C < 2, sigma not finite and
 * positive, a NULL pointer, boxes not 16-byte aligned.  DFQ_E_UNSUPPORTED: N * (C - 1) above INT32_MAX. */
int dfq_ssd_soft_nms(const float* scores, const float* boxes, int32_t* candidates, int32_t* counts, int64_t* offsets,
                     const DfqSsdNms* d, float sigma, void* stream);
/* The flat output of dfq_ssd_soft_nms's picks, laid out as dfq_ssd_compact lays out the hard picks (out_probs the picks'
 * decayed scores).  It runs the same soft NMS again on the same inputs, d and sigma, with candidates and offsets as
 * dfq_ssd_soft_nms left them, and writes each pick straight to its row.  Refusals of dfq_ssd_soft_nms, and DFQ_E_ARG for
 * a NULL output or out_boxes not 16-byte aligned. */
int dfq_ssd_soft_compact(const float* scores, const float* boxes, int32_t* candidates, const int64_t* offsets,
                         const float* image_sizes, float* out_boxes, int64_t* out_labels, float* out_probs,
                         const DfqSsdNms* d, float sigma, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Segmentation evaluation (utils/segmentation/utils.py forward_all, utils/metrics.py Evaluator) for a batch
 * ------------------------------------------------------------------------------------------- */
#define DFQ_SEG_LABEL_U8 0
#define DFQ_SEG_LABEL_I64 1
#define DFQ_SEG_LABEL_F32 2
typedef struct DfqSegArgmax {
  int32_t N, C, H, W;            /* logits fp32 NCHW [N, C, H, W], contiguous                                          */
  int32_t OH, OW;                /* output size: pred and labels are [N, OH, OW]                                       */
  int32_t align_corners;         /* 0 or 1; ignored when (OH, OW) == (H, W) (torch's plain copy)                       */
  int32_t label_type;            /* DFQ_SEG_LABEL_U8 (uint8), _I64 (int64) or _F32 (float32)                           */
} DfqSegArgmax;
/* Per output pixel (n, oh, ow): the C values of F.interpolate(logits, (OH, OW), mode="bilinear", align_corners) at that
 * pixel, bit for bit torch's CUDA upsample_bilinear2d (the plain copy when the size does not change), and their argmax
 * under torch's CUDA max(dim) rule: the first NaN wins over every number, otherwise the larger value, and on equal values
 * (-0.0 equal to +0.0) the lower index.  pred (int64 [N, OH, OW], optional) receives the argmax.  count (uint64 [C, C],
 * optional, accumulated: the caller clears it) receives, per pixel whose label gt passes the Evaluator's mask
 * 0 <= gt < C, one count at [gt][argmax].  The label of labels [N, OH, OW] is the value itself for uint8 and int64; for
 * float32 it is the value truncated toward zero (numpy's astype(np.uint8)) when -1 < v < 256, and NaN or any other value
 * is dropped.  labels and count are both given or both NULL; at least one of pred and count is given.
 * DFQ_E_ARG, with a reason and before any write: d NULL, a size below 1, align_corners not 0 or 1, an unknown label_type,
 * logits NULL, labels without count or count without labels, neither pred nor count, a pointer not aligned to its element
 * (labels to its label type), count or pred overlapping another buffer.  DFQ_E_UNSUPPORTED: C above 160, 2^62 elements
 * or more. */
int dfq_seg_argmax(const float* logits, const void* labels, int64_t* pred, uint64_t* count, const DfqSegArgmax* d,
                   void* stream);

/* ---------------------------------------------------------------------------------------------
 * Classification accuracy (main_cls.py inference_all), counted on the device
 * ------------------------------------------------------------------------------------------- */
/* Per row n of logits fp32 [N, C] (contiguous): the argmax of the row under torch's CUDA max(dim) rule (as
 * dfq_seg_argmax: the first NaN wins over every number, otherwise the larger value, and on equal values, -0.0 equal to
 * +0.0, the lower index).  pred (int64 [N], optional) receives it.  correct (uint64 [1], optional, accumulated: the caller
 * clears it) receives the number of rows whose label (labels int64 [N]) equals the argmax; a label outside 0 .. C-1
 * never does.  labels and correct are both given or both NULL; at least one of pred and correct is given.  Does not
 * synchronise.  DFQ_E_ARG, with a reason and before any write: N or C below 1, logits NULL, labels without correct or
 * correct without labels, neither pred nor correct, a pointer not aligned to its element, correct or pred overlapping
 * another buffer.  DFQ_E_UNSUPPORTED: 2^60 logits or more. */
int dfq_cls_count(const float* logits, const int64_t* labels, int64_t* pred, uint64_t* correct, int64_t N, int32_t C,
                  void* stream);

/* ---------------------------------------------------------------------------------------------
 * VOC average precision of SSD detections (main_ssd.py compute_average_precision_per_class,
 * utils/detection/measurements.py), accumulated batch by batch
 * ------------------------------------------------------------------------------------------- */
#define DFQ_MAP_IGNORED 0              /* verdict of a detection: neither true nor false positive (a difficult box) */
#define DFQ_MAP_TP 1
#define DFQ_MAP_FP 2
#define DFQ_MAP_ERR_DET_LABEL 1        /* bits of the device error word */
#define DFQ_MAP_ERR_GT_LABEL 2
#define DFQ_MAP_ERR_DET_OFFSETS 4
#define DFQ_MAP_ERR_GT_OFFSETS 8
/* One batch of N images: detections det_boxes fp32 [T, 4] (corner form, pixels), det_labels int64 [T], det_probs fp32 [T],
 * image n's rows det_offsets[n] .. det_offsets[n + 1] (int64 [N + 1]); ground truth gt_boxes fp32 [G, 4] (0-based corner
 * form, pixels), gt_labels int64 [G], gt_difficult uint8 [G] (non-zero: difficult), image n's rows gt_offsets[n] ..
 * gt_offsets[n + 1].  Adds each non-difficult box to gt_count[label] (uint64 [C], accumulated).  Per detection t of class
 * c: box = fl32(fl32(b + 1) - 1) per coordinate (the text round trip of main_ssd.py); no box of class c in the image:
 * false positive; else m = max and g = argmax of iou_of(box, gt) over the image's boxes of class c in annotation order
 * (box_utils' fp32 op order; the first NaN, else the first maximum); unless (double)m > iou_threshold: false positive;
 * box g difficult: ignored; else box g goes to the first detection claiming it in score-descending order (equal scores:
 * the lower row), a true positive, and every later claim is a false positive.  Writes keys[t] = (c << 32) | the score's
 * descending rank bits (-0.0 equal to +0.0, NaN last) and flags[t] = DFQ_MAP_IGNORED / _TP / _FP; pass keys and flags
 * offset to where the batch is appended.  Checks needing device data set bits of *error (atomicOr) instead of failing:
 * a detection label outside 1 .. C-1, a ground-truth label outside 0 .. C-1, offsets that do not run from 0 up to T
 * (resp. G) without decreasing; with bad offsets nothing of the batch is matched.  Does not synchronise.  DFQ_E_ARG, with a reason
 * and before any write: C < 2, N < 1, T or G < 0, a NULL pointer that is needed (the detection buffers when T > 0, the
 * ground-truth buffers when G > 0), boxes not 16-byte aligned.  DFQ_E_UNSUPPORTED: C above 4096, T above INT32_MAX. */
int dfq_map_match(const float* det_boxes, const int64_t* det_labels, const float* det_probs, const int64_t* det_offsets,
                  int64_t T, const float* gt_boxes, const int64_t* gt_labels, const uint8_t* gt_difficult,
                  const int64_t* gt_offsets, int64_t G, int32_t N, int32_t C, double iou_threshold, uint64_t* keys,
                  uint8_t* flags, uint64_t* gt_count, int32_t* error, void* stream);
/* The precision/recall curve of every class c = 1 .. C-1 over the D accumulated detections (keys, flags of
 * dfq_map_match), ordered by a stable sort on (class ascending, score descending): equal scores keep the order they were
 * appended in.  tp, fp the cumulative counts, precision = tp / (tp + fp), recall = tp / gt_count[c], float64.
 * use_2007 = 1: out[(c - 1) * 11 + k] = max(precision[recall >= k * 0.1]) (NaN-propagating), 0.0 when nothing is
 * selected, and term_count[c] (int64 [C]) = the class's number of detections; out_len >= 11 * (C - 1).  use_2007 = 0: the area terms (recall[j + 1] - recall[j]) * precision'[j + 1] of
 * compute_average_precision at each j where the padded recall changes, precision' the running maximum from the end
 * (NaN-propagating) of the padded precision; class c's terms, term_count[c] of them (int64 [C]), start at
 * (c - 1) + the sum of gt_count[1 .. c-1]; out_len >= G + C for G ground-truth boxes in all.  A class without non-difficult
 * ground truth (gt_count 0) yields values without meaning.  Does not synchronise.  DFQ_E_ARG, with a reason and before any
 * write: C < 2, D < 0, use_2007 not 0 or 1, a needed NULL pointer, out_len too small.  DFQ_E_UNSUPPORTED: C above 4096,
 * D above INT32_MAX. */
int dfq_map_curve(const uint64_t* keys, const uint8_t* flags, int64_t D, int32_t C, const uint64_t* gt_count,
                  int32_t use_2007, double* out, int64_t out_len, int64_t* term_count, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Evaluation preprocessing: the reference's resize, crop and normalisation of decoded uint8 images
 * (torchvision Resize + CenterCrop + ToTensor + Normalize, custom_transforms FixScaleCrop + Normalize,
 * SSD PredictionTransform), a batch of images of mixed sizes in one launch
 * ------------------------------------------------------------------------------------------- */
#define DFQ_PRE_PIL_BILINEAR 0   /* Pillow BILINEAR: 22-bit taps, both passes rounded and clipped to uint8          */
#define DFQ_PRE_CV_LINEAR 1      /* OpenCV INTER_LINEAR on uint8: 11-bit taps, int32 rows, the vectorised vertical step */
#define DFQ_PRE_NORM_F32 0       /* (float(u) / 255 - mean) / std, each step in fp32 (torchvision)                    */
#define DFQ_PRE_NORM_F64 1       /* float(u) / 255 in fp32; - mean and / std in fp64, each rounded to fp32 (numpy)     */
#define DFQ_PRE_NORM_SUB_DIV 2   /* (float(u) - mean) / std, each step in fp32 (SubtractMeans, / std)                 */
/* One image of the batch.  Offsets are bytes into the batch blob (one device buffer).  A tap table of an axis holds, per
 * output coordinate after the crop, K int32 pairs {source index, weight}; the source indices of each coordinate are
 * ascending, and so is the first and the last index from one coordinate to the next.  Pairs past a coordinate's own taps
 * repeat its last index with weight 0. */
typedef struct DfqPreImage {
  int64_t src;                   /* uint8 HWC RGB [H, W, 3], contiguous                                               */
  int64_t label;                 /* uint8 [H, W] label, or -1                                                         */
  int64_t xtap, ytap;            /* column and row tap tables: out_w * xk and out_h * yk pairs                        */
  int64_t xnear, ynear;          /* int32 source column / row of each label output, or -1 (with label -1)             */
  int32_t H, W;
  int32_t xk, yk;                /* taps per output column / row, 1 .. 4096                                           */
} DfqPreImage;
typedef struct DfqPreResample {
  int32_t n;                     /* images; out is float32 [n, 3, out_h, out_w], labels float32 [n, out_h, out_w]      */
  int32_t out_h, out_w;
  int32_t filter;                /* DFQ_PRE_PIL_BILINEAR or DFQ_PRE_CV_LINEAR                                         */
  int32_t norm;                  /* DFQ_PRE_NORM_*                                                                    */
  int32_t _pad;
  int64_t blob_bytes;            /* size of the blob: every table and image must lie inside it                        */
  float mean[3], std[3];         /* DFQ_PRE_NORM_F32 and _SUB_DIV                                                     */
  double mean64[3], std64[3];    /* DFQ_PRE_NORM_F64                                                                  */
} DfqPreResample;
/* Per output pixel (n, y, x) and channel c: the resized value through the taps of row y and column x (horizontal pass
 * first: Pillow rounds and clips it to uint8, OpenCV keeps the int32 sum), then the normalisation, written to out
 * [n, c, y, x].  With image n's label given, labels[n, y, x] = float(label[ynear[y], xnear[x]]).  images: host array of
 * d->n descriptors, uploaded by the call; blob: device pointer.  labels is NULL exactly when no image has a label.
 * DFQ_E_ARG, with a reason and before any launch: d, images, blob or out NULL, n, out_h or out_w below 1, an unknown
 * filter or norm, a std of zero, an image below 1 x 1, taps outside 1 .. 4096, a table or image outside the blob or
 * misaligned, labels given for some images only or without the labels pointer.  The tables' contents live on the device
 * and are not read by the call: every source index must lie in its image (columns below W, rows below H) and follow the
 * order stated above, or the kernel reads outside the image.  dfq_b200.preprocess builds them so. */
int dfq_pre_resample(const DfqPreResample* d, const DfqPreImage* images, const void* blob, float* out, float* labels,
                     void* stream);

/* ---------------------------------------------------------------------------------------------
 * JPEG decoding: baseline sequential Huffman streams (SOF0 / SOF1, 8-bit, 1 component or 3 YCbCr components with luma
 * sampling 1x1, 2x1 or 2x2 and chroma 1x1, one interleaved scan, any restart interval) decoded as libjpeg-turbo decodes
 * them with its defaults (jpeg_idct_islow, fancy upsampling, ycc_rgb_convert), into uint8 HWC RGB
 * ------------------------------------------------------------------------------------------- */
/* One Huffman table as libjpeg's jpeg_make_d_derived_tbl derives it: maxcode[l] the largest code of length l (-1 when
 * none, maxcode[17] 0xFFFFF), valoff[l] the index into vals of that length's first code minus the code, look[] the next
 * 9 bits -> (length << 8 | symbol) for codes of up to 9 bits, 0 otherwise. */
typedef struct DfqJpegHuff {
  int32_t maxcode[18];
  int32_t valoff[18];
  uint16_t look[512];
  uint8_t vals[256];
} DfqJpegHuff;
/* The tables of one stream, per component in frame order: the quantisation table in natural order and the scan's DC and
 * AC Huffman tables.  Gray streams use entry 0 only. */
typedef struct DfqJpegTables {
  int32_t q[3][64];
  DfqJpegHuff dc[3], ac[3];
} DfqJpegTables;
typedef struct DfqJpegImage {
  int64_t dst;                   /* uint8 HWC RGB [H, W, 3] output: byte offset in the blob                           */
  int64_t tables;                /* its DfqJpegTables: byte offset in the blob, 8-byte aligned                         */
  int32_t H, W;
  int32_t ncomp;                 /* 1 (gray, written as R = G = B) or 3 (YCbCr)                                        */
  int32_t hs, vs;                /* luma sampling: 1x1, 2x1 or 2x2 (1x1 for gray); chroma is 1x1                       */
  int32_t mcux, mcuy;            /* MCUs per row and per column: ceil(W / (8 hs)), ceil(H / (8 vs))                    */
  int32_t _pad;
} DfqJpegImage;
/* One restart interval of one image: its entropy-coded bytes (byte stuffing included, the RSTn marker and fill bytes
 * not), which decode MCUs mcu0 .. mcu0 + mcus - 1 with the DC predictors starting at zero. */
typedef struct DfqJpegSegment {
  int64_t begin, end;            /* byte offsets in the blob                                                           */
  int32_t image;
  int32_t mcu0, mcus;
  int32_t _pad;
} DfqJpegSegment;
typedef struct DfqJpegDecode {
  int32_t n, nseg;               /* images, segments: 1 .. 65535 images, 1 .. 2^31 - 1 segments                         */
  int64_t blob_bytes;            /* size of the blob: every segment, table block and output must lie inside it          */
  uint64_t call;                 /* tag of this call in the error word, below 2^31                                      */
} DfqJpegDecode;
#define DFQ_JPEG_BAD_CODE 1      /* error reasons, OR-ed into error[1]                                                 */
#define DFQ_JPEG_BAD_RUN 2
#define DFQ_JPEG_SHORT_SCAN 4
/* Decodes every image of the batch into its dst.  images, segs: host arrays, uploaded by the call; blob: device pointer.
 * error: device uint64 [2].  A segment found corrupt on the device (an invalid Huffman code, a run past coefficient 63,
 * data that ends before its last MCU) stops that segment's decode, atomicMin's (call << 32 | image) into error[0] and
 * OR's its reason into error[1]; that image's pixels are then unspecified, and no read or write leaves its segment, its
 * tables or its output.  Workspace (int16 coefficients and the component planes) is allocated stream-ordered and freed
 * by the call.  Does not synchronise.  DFQ_E_ARG, with a reason and before any launch: a NULL pointer, n or nseg out of
 * range, an image of unsupported geometry or whose MCU counts disagree with its size, a table block, output or segment
 * outside the blob, a segment whose image or MCUs are out of range, or segments that do not cover each image's MCUs
 * exactly once in order. */
int dfq_jpeg_decode(const DfqJpegDecode* d, const DfqJpegImage* images, const DfqJpegSegment* segs, void* blob,
                    uint64_t* error, void* stream);

/* ---------------------------------------------------------------------------------------------
 * PNG label decoding: non-interlaced 8-bit palette (indices, the palette never applied) or 8-bit gray streams, decoded
 * as Pillow's Image.open reads them (zlib inflate fed one row at a time, then the five scanline filters), into uint8 HW
 * ------------------------------------------------------------------------------------------- */
typedef struct DfqPngImage {
  int64_t src, src_end;          /* the zlib stream (its 2-byte header, the IDAT payloads joined): byte offsets in the blob */
  int64_t work;                  /* H * (W + 1) bytes of room for the filtered scanlines: byte offset in the blob          */
  int64_t dst;                   /* uint8 [H, W] output: byte offset in the blob                                           */
  int32_t H, W;
} DfqPngImage;
typedef struct DfqPngDecode {
  int32_t n;                     /* images, 1 .. 65535                                                                    */
  int32_t _pad;
  int64_t blob_bytes;            /* size of the blob: every stream, workspace and output must lie inside it               */
  uint64_t call;                 /* tag of this call in the error word, below 2^31                                        */
} DfqPngDecode;
#define DFQ_PNG_BAD_BLOCK 1      /* error reasons, OR-ed into error[1]: block type 3                                      */
#define DFQ_PNG_BAD_CODESET 2    /* an invalid code-length, literal/length or distance code set                           */
#define DFQ_PNG_BAD_CODE 4       /* an invalid literal/length or distance code                                            */
#define DFQ_PNG_FAR 8            /* a distance past the start of the output                                               */
#define DFQ_PNG_STORED_LEN 16    /* a stored block whose LEN and NLEN disagree                                            */
#define DFQ_PNG_SHORT 32         /* the stream ends before the last row, not at a row's end with its whole trailer       */
#define DFQ_PNG_BAD_FILTER 64    /* a scanline filter type above 4                                                        */
#define DFQ_PNG_ADLER 128        /* the Adler-32 after the last row's final block differs                                 */
/* Inflates each image's stream into its work room and unfilters the scanlines into its dst.  images: host array of d->n
 * descriptors, uploaded by the call; blob: device pointer; error: device uint64 [2].  Past the image's last byte the
 * stream is still decoded up to the first symbol that would write (block headers, code sets, end-of-block codes, a
 * distance code after a length, the Adler-32 after the final block), as zlib does for Pillow.  A final block that ends
 * at the end of an earlier row, followed by its whole and right Adler-32, leaves the rows not reached zero, as Pillow
 * does.  A stream found corrupt
 * stops that image, atomicMin's (call << 32 | image) into error[0] and OR's its reasons into error[1]; that image's
 * output is then unspecified, and no read or write leaves its stream, its work room or its output.  The zlib header is
 * not read: the caller checks it.  Does not synchronise.  DFQ_E_ARG, with a reason and before any launch: a NULL
 * pointer, n out of range, an image below 1 x 1 or above 2^31 - 1 pixels, a stream shorter than its header, or a
 * stream, work room or output outside the blob or overlapping one another. */
int dfq_png_decode(const DfqPngDecode* d, const DfqPngImage* images, void* blob, uint64_t* error, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DFQ_B200_H_ */
