/*
 * b200tip.h — C ABI of libb200tip.so, the H100 (sm_90a) scoring engine behind the
 * reference's `src.core` prioritizer API (testingautomated-usi/simple-tip).
 *
 * The reference has no FFI layer: its boundary is the Python class API of src/core
 * (SURVEY.md §8b).  The host mirror in simple_tip_b200/core keeps those classes and calls
 * the entry points below through ctypes.  Every array argument is a DEVICE pointer to a
 * contiguous row-major buffer owned by the caller (PyTorch on the Python side); the library
 * never frees caller memory and keeps no state between calls.  `stream` is a cudaStream_t
 * passed as void*; launches are asynchronous on it.  Every function returns 0 on success or
 * a negative tip_status; tip_last_error() returns a thread-local message.
 *
 * Which reference arithmetic each entry point replaces (paths relative to the reference):
 *   tip_deepgini        src/core/deepgini.py:31-35     argmax + 1 - sum(p*p)
 *   tip_softmax_stat    handler_model.py:23-85 uwiz MaxSoftmax / PredictionConfidenceScore / SoftmaxEntropy
 *                       (and DeepGini) on softmax outputs
 *   tip_vote_add        handler_model.py:148-166 uwiz VariationRatio: argmax votes of MC-dropout samples,
 *   tip_vote_finish     streamed pass by pass; mode and 1 - votes / samples
 *   tip_kmnc            src/core/neuron_coverage.py:82-94 (+ sum_score :8-22)
 *   tip_kmnc_packed     the same profile bit-packed in HBM, for tip_cam_bits
 *   tip_cam_buckets     src/core/prioritizers.py:16-45 (greedy loop of cam) on compact KMNC profiles
 *   tip_pair_prep       (new) operand packing for the tensor-core pass
 *   tip_nn_filter       src/core/surprise.py:638-647   the B x M x D difference/norm/min, as a
 *                       wgmma pass that yields a per-query candidate set provably containing
 *                       NumPy's argmin
 *   tip_nn_rerank       src/core/surprise.py:640-648   exact np.linalg.norm / np.min / np.argmin
 *                       on the candidates, in NumPy's summation order (bit-identical)
 *   tip_gather_rows     src/core/surprise.py:648       to_ats[closest_position]
 *   tip_whiten          scipy==1.4.1 gaussian_kernel_estimate: points . cholesky(inv_cov)
 *   tip_kde_lse         scipy==1.4.1 gaussian_kernel_estimate pair loop (called from
 *                       src/core/stable_kde.py:101), in the log domain
 *   tip_kde_combine     merge of per-column-chunk (max, sum) partials
 *   tip_kmeans_fit      src/core/surprise.py:117-118 KMeans(n_clusters=k, n_init, max_iter).fit (sklearn KMeans:
 *                       greedy k-means++ seeding + Lloyd iterations, all n_init runs in one kernel)
 *   tip_kmeans_predict  src/core/surprise.py:133 best_clusterer.predict (sklearn KMeans.predict), and the
 *                       final relabel / inertia of a fit
 *   tip_sil_prep        (new) operand packing of the silhouette pass
 *   tip_sil_dsum        src/core/surprise.py:119 silhouette_score: the all-pairs Euclidean distance sums
 *                       (sklearn pairwise_distances_chunked + np.bincount per cluster), as a wgmma pass
 *   tip_sil_finish      sklearn silhouette_samples: a, b, (b - a) / max(a, b), nan -> 0
 *   tip_gmm_quad        src/core/surprise.py:508-509,518 GaussianMixture.fit / score_samples (sklearn
 *                       _estimate_log_gaussian_prob, 'full': |X @ prec_chol - mu @ prec_chol|^2), fp64 DMMA
 *   tip_gmm_resp        sklearn _estimate_log_prob_resp (logsumexp, exp(log_resp)) and _e_step's mean
 *   tip_gmm_moments     sklearn _estimate_gaussian_parameters: nk = sum(resp) + 10 eps, means = resp.T @ X / nk
 *   tip_gmm_scatter     sklearn _estimate_gaussian_covariances_full: (resp_k * diff.T) @ diff / nk + reg_covar I
 *   tip_cov_location    src/core/surprise.py:385-386 EmpiricalCovariance().fit: location_ = X.mean(0) and
 *                       np.cov's float64 centring mean (the scatter reuses tip_gmm_scatter)
 *   tip_col_var         src/core/surprise.py:421,433 LSA's column selection: np.var(x, axis=0), bit for bit
 *   tip_whiten_dmma     scipy==1.4.1 gaussian_kernel_estimate: dataset . cholesky(inv_cov) for the training rows
 *                       of LSA's device fit, fp64 DMMA (the covariance reuses tip_gmm_scatter)
 *   tip_levenshtein     src/core/text_corruptor.py:282-309 TextCorruptor._calculate_distances: the all-pairs
 *                       polyleven.levenshtein matrix of the dictionary, bit-parallel (Myers / Hyyro)
 *   tip_tok_count       case_study_imdb.py:321-336 keras_preprocessing 1.1.2 text_to_word_sequence: words per text
 *   tip_tok_emit        ... each word's bytes (offset, length, text, hash) in Keras' iteration order
 *   tip_tok_vocab_table ... the vocabulary's hash table
 *   tip_tok_fit         Tokenizer.fit_on_texts: word_counts, first occurrences and word_docs
 *   tip_tok_lookup      Tokenizer.texts_to_sequences and pad_sequences, fused
 *   tip_corrupt_*       src/core/text_corruptor.py:311-508 TextCorruptor.corrupt: the split, MD5 seeds, NumPy's PCG64
 *                       draws and the four corruptions, string for string
 *   tip_keras_adam      case_study_*.py model.fit: Keras' Adam update of every parameter of a model, one launch
 *   tip_softmax_xent    ... categorical cross-entropy of the softmax output, its gradient and the accuracy count
 *   tip_softmax_xent_seg  ... the same head for M models trained in one stack, one segment of rows per model
 *   tip_stack_gather    ... one step's batch for every model of a stack, in one launch
 *   tip_mc_head         handler_model.py get_pred_and_uncertainty: MC-dropout samples of a model's dropout head
 *                       (dropout masks, dense layers and softmax) from its trunk activations, in one launch
 *   tip_mc_head_stack   the same for the M heads of a stack of models, one seed per model
 */
#ifndef B200TIP_H
#define B200TIP_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TIP_VERSION 200

typedef enum tip_status {
  TIP_OK = 0,
  TIP_ERR_INVALID = -1,    /* bad argument (shape, dtype, alignment) */
  TIP_ERR_CUDA = -2,       /* CUDA runtime / driver error, see tip_last_error() */
  TIP_ERR_UNSUPPORTED = -3 /* not an sm_90 device */
} tip_status;

typedef enum tip_dtype {
  TIP_F32 = 0,
  TIP_F64 = 1,
  TIP_BF16 = 2,
  TIP_I16 = 3,
  TIP_I32 = 4
} tip_dtype;

/* operand roles / packing modes for tip_pair_prep */
#define TIP_ROLE_QUERY 0 /* rows become accumulator rows (test traces / stage-2 winners) */
#define TIP_ROLE_TRAIN 1 /* rows become accumulator columns (training traces)         */

/* row selection for tip_nn_rerank */
#define TIP_RANGE_SAME_CLASS 0   /* columns [off[c], off[c+1])                      */
#define TIP_RANGE_OTHER_CLASSES 1 /* columns [0, off[c]) U [off[c+1], off[C])       */

/* One unit of work of the tensor-core pass: a tile of query rows (128 rows, see
 * tip_nn_filter_tile) x a span of train rows. */
typedef struct tip_work_item {
  int32_t q_row0;  /* first query row of the tile                                   */
  int32_t q_rows;  /* valid rows in the tile (1..tile); others are computed, not stored */
  int32_t col0;    /* first train row of the span                                   */
  int32_t col1;    /* one past the last train row of the span                       */
  int32_t slot;    /* tip_kde_lse: partial-result slot of this span; unused otherwise */
  int32_t reserved; /* flags: bit 0 = every query ignores the train rows of its own class
                     * (tip_nn_filter with q_class / class_off) */
} tip_work_item;

int tip_version(void);
const char* tip_last_error(void);
/* sm count and compute capability of the current device */
int tip_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* number of kernels this library has launched in this process (bench.py: gpu_launches) */
uint64_t tip_launch_count(void);

/* ---- DeepGini (deepgini.py:31-35) ----------------------------------------------------
 * probs: n x c (TIP_F32 or TIP_F64).  pred[n] = first argmax, gini[n] = 1 - sum(p*p) in the
 * input dtype, summed in NumPy's pairwise order (bit-identical to np.sum(p*p, axis=1)). */
int tip_deepgini(const void* probs, int dtype, int64_t n, int64_t c, int32_t* pred, void* gini,
                 void* stream);

/* ---- uncertainty quantifiers of uncertainty-wizard 0.2.0 (handler_model.py:23-85,102-173) -----
 * tip_softmax_stat: probs n x c (TIP_F32 or TIP_F64); pred[n] = first argmax, out[n] in the input dtype:
 *   TIP_STAT_GINI     1 - sum(p*p), the same as tip_deepgini
 *   TIP_STAT_MAX      max(p)                                        MaxSoftmax
 *   TIP_STAT_PCS      top-1 minus top-2 of p (0 for a repeated max) PredictionConfidenceScore; needs c >= 2
 *   TIP_STAT_ENTROPY  -sum(q*log2(q)), q = p with exact zeros replaced by 1e-20   SoftmaxEntropy
 * GINI, MAX and PCS are bit-identical to NumPy; ENTROPY sums in NumPy's pairwise order, its log2 is within an
 * ulp of libm's.  The values are uncertainties or confidences as the quantifier defines them, unsigned.
 *
 * tip_vote_add: the argmax (first index) of every sampled row, added to counts[n x c] (int32, zeroed by the
 * caller before the first call).  Sample s of row i is the c-vector at probs + i*row_stride + s*sample_stride
 * (elements); dense [n, samples, c] input is sample_stride = c, row_stride = samples*c.  Calls accumulate, so
 * samples may arrive in chunks (MC-dropout passes).
 * tip_vote_finish: pred[n] = the lowest class with the most votes (scipy.stats.mode), vr[n] = 1 - votes/samples
 * (float64)                                                        VariationRatio */
#define TIP_STAT_GINI 0
#define TIP_STAT_MAX 1
#define TIP_STAT_PCS 2
#define TIP_STAT_ENTROPY 3
int tip_softmax_stat(const void* probs, int dtype, int64_t n, int64_t c, int kind, int32_t* pred, void* out,
                     void* stream);
int tip_vote_add(const void* probs, int dtype, int64_t n, int64_t c, int64_t samples, int64_t sample_stride,
                 int64_t row_stride, int32_t* counts, void* stream);
int tip_vote_finish(const int32_t* counts, int64_t n, int64_t c, int64_t samples, int32_t* pred, double* vr,
                    void* stream);

/* ---- KMNC (neuron_coverage.py:65-94) -------------------------------------------------
 * act: n x d (TIP_F32/TIP_F64); mins, jumps: d values of stat_dtype, jumps = (max-min)/k
 * computed by the caller with the reference's NumPy expression.  Thresholds are
 * t_i = min + jumps*i evaluated on the fly in stat_dtype (same rounding as NumPy).
 * bucket[n*d] (TIP_I16 or TIP_I32) = the i with t_i <= a < t_{i+1}, or -1; score[n] = number of
 * neurons with a bucket (== sum of the reference's dense profile). bucket may be NULL. */
int tip_kmnc(const void* act, int act_dtype, int64_t n, int64_t d, const void* mins,
             const void* jumps, int stat_dtype, int32_t sections, void* bucket, int bucket_dtype,
             int32_t* score, void* stream);
/* The same sections, bit-packed for tip_cam_bits (the reference's dense n x d x sections profile,
 * plane by plane): bits[n * sections * W] with W = tip_cover_packed_words(d).  Row r holds `sections`
 * planes of W words; in plane s, bit l of word 4g + i is set when neuron 128g + 4l + i lies in section
 * s — the layout of tip_cover_threshold (one plane: NAC's, two: NBC's plane order).  Padding bits are
 * 0; every word of a row is written.  score[n] as tip_kmnc.  Section membership is tip_kmnc's
 * arithmetic, so the bits are set exactly where tip_kmnc's bucket ids say. */
int tip_kmnc_packed(const void* act, int act_dtype, int64_t n, int64_t d, const void* mins,
                    const void* jumps, int stat_dtype, int32_t sections, uint32_t* bits, int32_t* score,
                    void* stream);

/* ---- Coverage-Additional Method over compact coverage profiles (prioritizers.py:16-59) ----
 * bucket: n x d section ids as tip_kmnc writes them (TIP_I16 / TIP_I32, -1 = none): the one-hot-per-
 * neuron profile of neuron_coverage.py:82-94 without its dense n x d x sections form.  Runs up to
 * `rounds` rounds of the reference's greedy loop — pick = first index of the largest gain (np.argmax),
 * mark the cells the pick newly covers, subtract from every sample the number of those cells it shares
 * — and stops for good when the best gain is 0.  Caller-owned state, all on the device:
 *   gain[n]      in: number of valid cells per sample (= KMNC score); updated in place
 *   covered      ceil(d*sections/32) words, zero before the first call
 *   newlist      2*d int32 scratch
 *   order[n]     out: the picks in order; state[0] = how many (zero before the first call)
 *   state[4]     {picks, done flag, scratch, scratch}, zero before the first call; call again with the
 *                same buffers while state[1] == 0 && state[0] < n.
 * The tail of the reference's generator (not-yet-picked samples by np.argsort(-scores), :47-59) is host
 * NumPy, so ties fall exactly as in the reference. */
int tip_cam_buckets(const void* bucket, int bucket_dtype, int64_t n, int64_t d, int32_t sections,
                    int32_t* gain, uint32_t* covered, int32_t* newlist, int32_t* order, int32_t* state,
                    int32_t rounds, void* stream);

/* ---- Surprise-coverage CAM (handler_surprise.py:101-115, prioritizers.py:16-45) ---------------------
 * The greedy picks of cam(values, SurpriseCoverageMapper.get_coverage_profile(values)) without the n x sections
 * profile.  thresholds: sections + 1 float64 values on the device, NaN-free and non-decreasing (the caller checks;
 * then every profile row has at most one True and the picks are the first sample of every non-empty bucket, in
 * ascending sample order).  values: n values of TIP_F32 (compared after exact widening to float64, NumPy's
 * promotion) or TIP_F64; sample i lies in bucket b when thresholds[b] <= v < thresholds[b+1]; NaN lies in none.
 * first[sections] uint32 scratch (reset here); out: order[0..count) = the picks, count[1] int32.
 * 1 <= sections <= TIP_SC_CAM_MAX_SECTIONS (one block ranks the buckets in shared memory), 0 <= n < 2^31. */
#define TIP_SC_CAM_MAX_SECTIONS 4096
int tip_sc_cam(const void* values, int dtype, int64_t n, const double* thresholds, int32_t sections,
               uint32_t* first, int32_t* order, int32_t* count, void* stream);

/* ---- sibling coverage criteria and their fit step (neuron_coverage.py:52-62,97-173;
 * aggregate_statistics.py:37-67 + welford==0.2.5) ------------------------------------------
 * tip_cover_threshold: act n x d (TIP_F32/TIP_F64); mode
 *   TIP_COVER_NAC   profile[n,d]   = act >  threshold                      (lo = hi = NULL)
 *   TIP_COVER_SNAC  profile[n,d]   = act >= hi[d]
 *   TIP_COVER_NBC   profile[n,d,2] = (act <= lo[d], act >= hi[d])
 * lo / hi: d boundaries of stat_dtype, computed by the caller with the reference's NumPy expressions
 * (min - s*std, max + s*std); comparisons run in NumPy's promoted dtype of (act, boundary), so the
 * profile is bit-identical.  profile_u8 (one byte per entry: the reference's dense bool array) and
 * bits (the same profile bit-packed for tip_cam_bits, tip_cover_packed_words(d) words per row and
 * plane, NBC: 2 planes; layout in csrc/coverage.cu) are both optional; score[n] = number of set
 * entries per sample (== sum_score, neuron_coverage.py:8-22). */
#define TIP_COVER_NAC 0
#define TIP_COVER_SNAC 1
#define TIP_COVER_NBC 2
int64_t tip_cover_packed_words(int64_t d);
int tip_cover_threshold(const void* act, int act_dtype, int64_t n, int64_t d, const void* lo,
                        const void* hi, int stat_dtype, double threshold, int mode, void* profile_u8,
                        uint32_t* bits, int32_t* score, void* stream);
/* Top-k neuron coverage of ONE layer (neuron_coverage.py:160-168): for every sample the k largest of its
 * d_layer activations are marked in profile_u8[r * row_stride + col_off + i] (all entries of the layer's
 * columns are written) and/or OR-ed into the packed words of neuron col_off + i (bits must be zero-filled
 * by the caller; bit_words = words per row).  k >= 0 is the number of neurons marked: the caller passes
 * len(range(d_layer)[-top_neurons:]), the count the reference's slice `argsort(layer)[..., -top_neurons:]`
 * takes (d_layer for top_neurons = 0, d_layer - |top_neurons| for negative values); k >= d_layer marks the
 * whole layer without running the k block-wide selection rounds.  Equal values: the higher index wins, NaN
 * ranks above everything (a stable ascending argsort's last entries; NumPy's unstable argsort leaves ties
 * implementation-defined). */
int tip_tknc(const void* act, int dtype, int64_t n, int64_t d_layer, int32_t k, void* profile_u8,
             int64_t row_stride, int64_t col_off, uint32_t* bits, int64_t bit_words, void* stream);
/* Streaming per-neuron statistics over a batch of n samples x d neurons: mins/maxs and welford==0.2.5's
 * `add` applied sample by sample in the activation dtype (mean, m2 = sum of squared deviations; the caller
 * keeps the integer count: count_before = samples folded in so far).  State arrays hold d values of
 * `dtype`; initial state: mean = m2 = 0, mins = +inf, maxs = -inf. */
int tip_stats_update(const void* act, int dtype, int64_t n, int64_t d, int64_t count_before, void* mean,
                     void* m2, void* mins, void* maxs, void* stream);

/* ---- Coverage-Additional Method over dense boolean profiles, bit-packed (prioritizers.py:16-45) ----
 * tip_pack_bool: byte profile n x f (non-zero = covered) -> ceil(f/32) words per row.
 * tip_cam_bits: bits n x words (any packing, the order of the picks does not depend on it).  One
 * persistent cooperative kernel runs up to max_rounds greedy rounds: pick = first index of the largest
 * gain, new = profile[pick] & ~covered, gain[i] -= popcount(profile[i] & new); it stops for good when
 * the best gain is 0.  Caller-owned device state: gain[n] (init_gain != 0: initialised here to the row
 * popcounts), covered2[2*words] zero-filled, cand_scratch[4*TIP_CAM_MAX_BLOCKS] int32, order[n],
 * state[4] = {picks, done, -, -} zero-filled before the first call; call again with the same buffers
 * (init_gain = 0) while state[1] == 0 && state[0] < n.  max_rounds must be even when more calls follow
 * (the covered set is double-buffered by round parity). */
#define TIP_CAM_MAX_BLOCKS 1024
int tip_pack_bool(const void* profile_u8, int64_t n, int64_t f, uint32_t* bits, void* stream);
int tip_cam_bits(const uint32_t* bits, int64_t n, int64_t words, int32_t* gain, uint32_t* covered2,
                 int32_t* cand_scratch, int32_t* order, int32_t* state, int32_t max_rounds,
                 int32_t init_gain, void* stream);
/* tip_cam_bits_stack: tip_cam_bits on the profiles of `models` models at once (a stack's), with one leading
 * model axis on every buffer but the scratch: bits [models, n, words], gain [models, n], covered2
 * [models, 2, words] zero-filled, order [models, n], state [models, 4] = {picks, done, -, -} per model,
 * cand_scratch as for tip_cam_bits.  Slice m of order and state equals tip_cam_bits on bits[m].  Call again
 * with the same buffers (init_gain = 0) while any model has done == 0 && picks < n; max_rounds must be even
 * when more calls follow.  models * n < 2^31.  More models than one co-resident grid holds run in consecutive
 * launches. */
int tip_cam_bits_stack(const uint32_t* bits, int64_t models, int64_t n, int64_t words, int32_t* gain,
                       uint32_t* covered2, int32_t* cand_scratch, int32_t* order, int32_t* state,
                       int32_t max_rounds, int32_t init_gain, void* stream);

/* ---- operand packing for the tensor-core pass ----------------------------------------
 * Packed row (bf16), D16 = round_up(d,16), one 16-wide tail block:
 *   segments == 1:  [ s*h(v) | tail ]                 v = fl32(x - center)
 *   segments == 3:  query: [ h | l | h | tail ]       h = bf16(v), l = bf16(v - h)
 *                   train: [ s*h | s*h | s*l | tail ]
 *   tail(query) = [1,1,1,0...]; tail(train) = bf16 3-way split of norm_coef*|v|^2
 * so that one K-loop accumulates  norm_coef*|y|^2 + s * <x, y>  in fp32.
 * sqnorm[rows] receives |h(v)|^2 (segments==1) or |v|^2 (segments==3) as fp32.
 * rounderr[rows] (may be NULL) receives the Euclidean norm of what the packed operand drops,
 * |v - h(v)| (segments==1) or |v - h - l| (segments==3), rounded up: the per-row input-rounding
 * term of tip_nn_filter's error window.
 * tip_pair_pitch returns the packed row pitch in elements (multiple of 64). */
int64_t tip_pair_pitch(int64_t d, int segments);
int tip_pair_prep(const void* src, int dtype, int64_t rows, int64_t d, const float* center,
                  int role, int segments, float scale, float norm_coef, void* dst_bf16,
                  float* sqnorm, float* rounderr, void* stream);

/* Query side of tip_nn_filter in one launch: packs the queries (segments = 1, no scaling) and
 * resets the per-query filter state (row_min_bits = +inf, cand_cnt = 0).  q_idx (may be NULL): packed row r is
 * taken from q + q_idx[r]*d — the class-sorting gather of DSA.__call__ (surprise.py:580-587) fused into the pack. */
int tip_nn_query_prep(const void* q, int dtype, int64_t m, int64_t d, const float* center,
                      void* q_pack, float* q_sqnorm, float* q_rounderr, uint32_t* row_min_bits,
                      int32_t* cand_cnt, const int32_t* q_idx, void* stream);

/* ---- nearest-neighbour candidate filter (wgmma + TMA) ------------------------------
 * q_pack: m x pitch, t_pack: n x pitch (tip_pair_prep, scale=-2, norm_coef=1).
 * For every query row and every work item covering it, scans the item's train span and
 * appends one entry per 32-row chunk of train rows that contains a row whose approximate squared
 * distance is within the proven error window of the running minimum (see DESIGN.md §4):
 * cand_idx[(row*cap + k)*2] = first train row of the chunk, cand_idx[(row*cap + k)*2 + 1] = 32-bit
 * mask of the rows of the chunk that pass (cand_idx holds 2*cap int32 per query); cand_cnt[row]
 * counts appends (may exceed cap: overflow -> tip_nn_rerank falls back to an exact scan).
 * row_min_bits[m] (uint32 float bits, initialised to +inf = 0x7f800000 by the caller) carries
 * the running minimum across items/CTAs.  t_rmax = max_j |h(y_j)| over the train rows.
 * q_rounderr[m] / t_errmax = max_j rounderr(y_j) (tip_pair_prep) give the window its measured
 * input-rounding term |d_bf16 - d| <= rounderr(x) + rounderr(y); with q_rounderr == NULL the
 * a-priori bound 2^-9 (|h(x)| + |h(y)|) is used instead (about twice as wide).
 * Scheduling: CTA b of the G = min(n_items, #SMs) persistent CTAs runs items b, b + G, ... below
 * n_static; items [n_static, n_items) are a shared pool that CTAs drain through sched_counter
 * once their static share is done — the pool evens out CTAs whose
 * tiles turn out slower.  sched_counter points to TWO int32 that are zero on entry; the kernel
 * leaves them zero (one call at a time per counter pair).  n_static == n_items (sched_counter may
 * be NULL) is a purely static run;
 * pools need the resident-query kernel (d <= 128).  Items with col0 == col1 are skipped.
 * q_class[m] / class_off[C+1] (may be NULL if no item sets flag bit 0): for flagged items a query of
 * class c ignores train rows [class_off[c], class_off[c+1]) — DSA's other-class search over
 * query tiles that mix classes (surprise.py:622-629). */
int tip_nn_filter(const void* q_pack, const float* q_sqnorm, int64_t m, const void* t_pack,
                  int64_t n, int64_t d, int64_t pitch, const tip_work_item* items,
                  int32_t n_items, const int32_t* q_class, const int32_t* class_off, float t_rmax,
                  const float* q_rounderr, float t_errmax, uint32_t* row_min_bits, int32_t* cand_idx,
                  int32_t* cand_cnt, int32_t cap, int32_t n_static, int32_t* sched_counter,
                  void* stream);

/* tip_nn_filter whose queries end per class at a bound known only on the device (DSA's stage 2 on distinct
 * winners, tip_dsa_distinct_winners): q_live_end[m] (may be NULL: tip_nn_filter) holds, for every query row, one
 * past the last row that holds a query in its class's range.  An item covers rows [q_row0, min(q_row0 + q_rows,
 * q_live_end[q_row0])) of its tile; an item without such rows is skipped when it is drawn (no query-tile load, no
 * pipeline stage), so a work list that draws its items through sched_counter (n_static == 0), ordered so that the
 * rows likeliest to be live come first, keeps the CTAs balanced whatever the live counts turn out to be. */
int tip_nn_filter_live(const void* q_pack, const float* q_sqnorm, int64_t m, const void* t_pack,
                       int64_t n, int64_t d, int64_t pitch, const tip_work_item* items,
                       int32_t n_items, const int32_t* q_class, const int32_t* class_off, float t_rmax,
                       const float* q_rounderr, float t_errmax, uint32_t* row_min_bits, int32_t* cand_idx,
                       int32_t* cand_cnt, int32_t cap, int32_t n_static, int32_t* sched_counter,
                       const int32_t* q_live_end, void* stream);

/* Tile geometry tip_nn_filter uses for traces of width d: work items must start on query rows
 * that are multiples of nothing in particular but cover at most *q_rows rows (192 for the resident-query
 * kernel, 128 for the streaming one); *t_rows is the train-tile height (128), useful for sizing spans. */
int tip_nn_filter_tile(int64_t d, int32_t* q_rows, int32_t* t_rows);
/* which tensor-core kernel tip_nn_filter runs for traces of width d: 1 = resident-query (d <= 128: the query
 * tile is loaded once per work item; 192 x 128 tiles), 0 = streaming (query and train chunks through one
 * ring; 128 x 128 tiles).  tip_kde_tile_rows: query rows per work item of tip_kde_lse*. */
int tip_nn_filter_kind(int64_t d);
int tip_kde_tile_rows(void);
int tip_kde_slot_parts(void);   /* partial (max, sum) pairs per work-item slot: part_max / part_sum hold slots x this x m */

/* ---- exact re-rank (NumPy-order distances, first-occurrence argmin) -------------------
 * q, t: original-dtype (TIP_F32/TIP_F64) matrices m x d and n x d; train rows are grouped by
 * class (class_off[C+1]); q_class[m] gives each query's class, mode the column range.
 * Rows with 1..cap candidate entries (tip_nn_filter's chunk + mask pairs, rows clipped to the
 * class range) are re-ranked over the flagged rows; rows with 0 or > cap
 * candidates (or cand_cnt == NULL) are scanned exhaustively over their range.
 * out_dist[m] (dtype) = sqrt(pairwise_sum((x-y)^2)) of the winner, out_pos[m] = its train row
 * (ties: lowest t_gid); optional out_gid[m] = t_gid of the winner (-1 if none) and
 * out_rows[m x d] = a copy of the winning train rows (DSA's stage-2 queries, surprise.py:648).
 * work: scratch of tip_nn_rerank_work_bytes(m, dtype) bytes (queue of queries that need the
 * exhaustive scan + the per-slice partial winners of that scan).  The caller zero-fills it once;
 * every call leaves the two words it relies on (queue length work[0], completion counter
 * work[1 + m]) at zero again, so the buffer can be reused by the next call on the same stream.
 * stats[0] += rows that took the exhaustive scan (stats[1] is reserved; candidate counts are in
 * cand_cnt).
 * next_*: optional (all NULL, or pack + sqnorm + row_min_bits + cand_cnt given): the winning rows are
 * also emitted as the packed queries and reset filter state of a following tip_nn_filter call —
 * exactly what tip_nn_query_prep(out_rows, center = next_center) would write — so DSA's second
 * stage (whose queries are stage 1's winners, surprise.py:627-629) needs no pack launch.
 * extras (optional, host struct read at launch time):
 * q_idx: the queries are rows q_idx[r] of q (no separately gathered copy needed); fin_*: fused result scatter.
 * next_seed_ub (optional, with next_rounderr): n floats, for every train row an upper bound on its exact
 * distance to SOME row the next search will scan for it (e.g. its nearest other-class row inside a fixed sample
 * of the training set, computed once at fit time; +inf = none).  The winner's bound, widened by the filter's own
 * error terms (next_t_rmax / next_t_errmax = the t_rmax / t_errmax of the next tip_nn_filter call), becomes the
 * initial next_row_min_bits instead of +inf: the next filter collects no far-away candidates while its running
 * minima warm up.  A seed never narrows the proven window below the final one (DESIGN.md §4). */
typedef struct tip_rerank_extras {
  const int32_t* q_idx;       /* query row r is q + q_idx[r]*d (e.g. class-sorted order over the caller's buffer) */
  const float* next_seed_ub;  /* see above */
  float next_t_rmax;
  float next_t_errmax;
  const void* fin_dist_a;     /* fused result scatter: with fin_out != NULL this search's distance is taken as dist_b */
  const int32_t* fin_gid;     /* and out[0..3][fin_idx[r]] = dist_a, dist_b, gid, dist_a / dist_b as tip_dsa_pack_out */
  const int32_t* fin_idx;     /* writes them (fin_idx == NULL: r itself); fin_dist_a in `dtype`, fin_out 4*fin_n_total */
  int64_t fin_n_total;        /* doubles */
  double* fin_out;
  int32_t count_overflow_only; /* != 0 (filtered searches only): queries whose candidate list is empty or overflowed are */
  int32_t reserved;            /* only COUNTED in work[0] — no queue, no exhaustive-scan launch, their outputs are not    */
                               /* written; the caller checks work[0] after the call, resets it and repeats without this   */
                               /* flag if it is non-zero (speculative execution of the normal, fallback-free case)        */
} tip_rerank_extras;
int32_t tip_sizeof_rerank_extras(void);   /* bindings check their struct layout against this */
int64_t tip_nn_rerank_work_bytes(int64_t m, int dtype);
int tip_nn_rerank(const void* q, const void* t, int dtype, int64_t m, int64_t n, int64_t d,
                  const int32_t* cand_idx, const int32_t* cand_cnt, int32_t cap,
                  const int32_t* q_class, const int32_t* class_off, int32_t n_classes, int mode,
                  const int32_t* t_gid, void* out_dist, int32_t* out_pos, int32_t* out_gid,
                  void* out_rows, int32_t* work, int64_t* stats, const float* next_center,
                  void* next_pack, float* next_sqnorm, float* next_rounderr,
                  uint32_t* next_row_min_bits, int32_t* next_cand_cnt, const tip_rerank_extras* extras,
                  void* stream);

/* DSA's stage 2 once per distinct stage-1 winner (its result depends on the winning train row alone,
 * surprise.py:622-631).  pos[m]: stage-1 winner positions (tip_nn_rerank's out_pos) of class-sorted inputs whose
 * class ranges are q_off[C+1] (device); class_off[C+1] (device) as for tip_nn_rerank, every class at most
 * max_class_rows rows (tip_dsa_distinct_smem_bytes(max_class_rows) <= 48 KB).  Class c's slots are
 * [q_off[c], q_off[c] + k[c]): its distinct winners in ascending train-row order, then one slot for its inputs without
 * a winner (pos outside the class: a zero row is searched, as tip_nn_rerank's next_* packs it) if it has any.  For
 * every slot s below the bound: rows[s] = the winner's train row (dtype, m x d), the packed stage-2 query state
 * (what tip_nn_rerank's next_* with next_seed_ub = seed_ub writes for that row) and slot_class[s] = c; past it
 * slot_class[s] = -1 (tip_nn_rerank writes "no row" there), cand_cnt[s] = 0 and the rest of the state is not
 * written.  live_end[s] = q_off[c] +
 * k[c] for every slot of class c (tip_nn_filter_live), slot[i] = the slot of input i.  blocks_per_class blocks share
 * each class's slots.  Nothing is kept between calls. */
int64_t tip_dsa_distinct_smem_bytes(int64_t max_class_rows);
int tip_dsa_distinct_winners(const int32_t* pos, int64_t m, const int32_t* q_off, const int32_t* class_off,
                             int32_t n_classes, int64_t max_class_rows, int32_t blocks_per_class, const void* t,
                             int dtype, int64_t d, const float* center, const float* seed_ub, float t_rmax,
                             float t_errmax, void* rows, void* q_pack, float* q_sqnorm, float* q_rounderr,
                             uint32_t* row_min_bits, int32_t* cand_cnt, int32_t* slot_class, int32_t* live_end,
                             int32_t* k, int32_t* slot, void* stream);
/* dist_b[i] = slot_dist[slot[i]] for i < m; with out != NULL also the result scatter of tip_dsa_pack_out
 * (dist_a, that dist_b, gid, dist_a / dist_b into column idx[i] of out[4 x n_total]). */
int tip_dsa_slot_out(const void* slot_dist, int dtype, const int32_t* slot, int64_t m, const void* dist_a,
                     const int32_t* gid, const int32_t* idx, int64_t n_total, void* dist_b, double* out,
                     void* stream);

/* DSA result packing (surprise.py:576-611 scatter by index): for i < m,
 *   out[0*n_total + j] = dist_a[i], out[1*n_total + j] = dist_b[i], out[2*n_total + j] = gid[i],
 *   out[3*n_total + j] = dist_a[i] / dist_b[i]  (IEEE division in `dtype`, surprise.py:595)
 * with j = idx[i] (idx == NULL: j = i); values in `dtype` (TIP_F32/TIP_F64) are widened to double
 * exactly, gid (int32) likewise.  out holds 4*n_total doubles; columns not named by idx are left
 * untouched. */
int tip_dsa_pack_out(const void* dist_a, const void* dist_b, int dtype, const int32_t* gid,
                     const int32_t* idx, int64_t m, int64_t n_total, double* out, void* stream);

/* dst[i,:] = src[pos[i],:]  (rows of `row_bytes` bytes; pos < 0 -> zero row) */
int tip_gather_rows(const void* src, int64_t row_bytes, const int32_t* pos, int64_t m, void* dst,
                    void* stream);

/* ---- N_train sharded over the GPUs of one NVSwitch box (SURVEY.md 8e; no counterpart in the
 * reference — the dependency that forces the exchange is src/core/surprise.py:615-631: stage 2's
 * queries are the GLOBAL stage-1 winners) -------------------------------------------------------
 * A tip_comm is a set of symmetric receive buffers, one per rank (one process per GPU), opened
 * across processes through CUDA IPC.  An exchange is: every rank pushes m 16-byte records into the
 * slots of all peers with plain NVLink stores and raises a flag (tip_comm_push_*); the consumer
 * kernel (tip_shard_winner_queries / tip_comm_min / tip_comm_lse) waits for all flags and reduces the
 * `world` records per query from local memory in its prologue.  Exchanges must be issued in the same
 * order on every rank; at most `cap_records` records per exchange.  Set-up (host side, once):
 *   tip_comm_alloc      cudaMalloc + zero the local buffer, return its 64-byte IPC handle
 *   (all-gather the handles with torch.distributed)
 *   tip_comm_open       map the peers' buffers; all_handles = world x 64 bytes in rank order
 *   tip_comm_close      unmap the peers;  tip_comm_free_local frees the local buffer. */
#define TIP_COMM_MAX_WORLD 16
#define TIP_COMM_HANDLE_BYTES 64
typedef struct tip_comm tip_comm;
int64_t tip_comm_bytes(int32_t world, int64_t cap_records);
int tip_comm_alloc(int32_t world, int64_t cap_records, void** local_buf, void* ipc_handle);
int tip_comm_open(int32_t rank, int32_t world, void* local_buf, const void* all_handles,
                  int64_t cap_records, tip_comm** out);
int tip_comm_close(tip_comm* comm);
int tip_comm_free_local(void* local_buf);
/* record i = (bit pattern of dist[i] (NaN = no row on this shard), gid[i] or 0): the per-shard result
 * of tip_nn_rerank for query i; dtype TIP_F32 / TIP_F64 */
int tip_comm_push_nn(tip_comm* comm, const void* dist, int dtype, const int32_t* gid, int64_t m,
                     void* stream);
/* record i = this shard's partial KDE sum (running max, sum of exp(. - max)) of tip_kde_combine */
int tip_comm_push_lse(tip_comm* comm, const float* part_max, const float* part_sum, int64_t m,
                      void* stream);
/* out_dist[i] = min over the ranks of the pushed distances (NaN if no shard had a row) */
int tip_comm_min(tip_comm* comm, int dtype, int64_t m, void* out_dist, void* stream);
/* merged log-sum-exp partials, in rank order, identical on every rank: out_max = max_r max_r,
 * out_sum = sum_r sum_r * exp(max_r - out_max) (double) */
int tip_comm_lse(tip_comm* comm, int64_t m, float* out_max, double* out_sum, void* stream);
/* Global stage-1 winners -> stage-2 queries.  comm != NULL: waits for the exchange started by the
 * last tip_comm_push_nn and takes, per query, the lexicographic minimum of (distance, original
 * index) over the shards; comm == NULL: gdist[m] / ggid[m] hold that minimum already (reduced by
 * torch.distributed).  train_full: the whole (post-subsample) training set, n_full x d in the trace
 * dtype, rows in ORIGINAL order, replicated on every rank (C5: 10.5 GB of 180).  Writes the global
 * dist_a (NaN if the class has no training row anywhere), the winner's original index (-1), a copy
 * of the winning rows (out_rows, m x d: the exact re-rank's queries) and the packed bf16 queries +
 * reset filter state of the following tip_nn_filter call (see tip_nn_rerank's next_* outputs). */
int tip_shard_winner_queries(tip_comm* comm, const void* gdist, const int32_t* ggid, int dtype,
                             int64_t m, int64_t d, const void* train_full, int64_t n_full,
                             const float* center, void* out_dist, int32_t* out_gid, void* out_rows,
                             void* next_pack, float* next_sqnorm, float* next_rounderr,
                             uint32_t* next_row_min_bits, int32_t* next_cand_cnt, void* stream);

/* ---- LSA: whitening and the fused Gaussian-KDE log-sum-exp ---------------------------
 * out[m x d_out] (fp32) = (x[:, cols] - mu) . w, x: m x d_in (TIP_F32/TIP_F64), cols[d_out] the kept
 * columns (NULL = all), mu: d_out doubles, w: d_out x d_out fp32 row-major. */
int tip_whiten(const void* x, int dtype, int64_t m, int64_t d_in, const int32_t* cols,
               int64_t d_out, const double* mu, const float* w, float* out, void* stream);

/* out[m] (double) = sum_k y[row,k]^2 of a whitened matrix y (m x d fp32, from tip_whiten): the squared
 * Mahalanobis distance to one centre (MDSA, surprise.py:374-393: sklearn EmpiricalCovariance.mahalanobis) or
 * the quadratic form of one mixture component (MLSA, surprise.py:498-520: sklearn
 * _estimate_log_gaussian_prob, y = (x - mu_k) . precisions_cholesky_k). */
int tip_row_sqnorm(const float* y, int64_t m, int64_t d, double* out, void* stream);

/* q_pack / t_pack from tip_pair_prep(segments=3, scale=1, norm_coef=-0.5 on the train side).
 * For every work item writes the partial (max_i a_ij, sum_i exp(a_ij - max)) of
 * a_ij = <p_i, q_j> - |p_i|^2/2 over the item's span into part_max/part_sum[(P*slot+h)*m + row],
 * P = tip_kde_slot_parts() (1: one row's columns are reduced in one place), h = 0..P-1 (so P*slots*m floats
 * each, which the caller initialises to -inf / 0). */
int tip_kde_lse(const void* q_pack, int64_t m, const void* t_pack, int64_t n, int64_t d,
                int64_t pitch, const tip_work_item* items, int32_t n_items, float* part_max,
                float* part_sum, void* stream);
/* The same pass with ONE fp16 segment (a third of the tensor work): operands from tip_pair_prep_f16, i.e.
 * a_ij = <h(p_i), h(q_j)> - |p_i|^2/2 with h = fp16 rounding (11-bit significands: |error| ~ 2^-12 per product,
 * against ~2^-17 for the three-segment bf16 form).  Whether that is accurate enough for rtol 1e-4 on the
 * log-density depends on the data; the caller verifies it against tip_kde_lse on a sample of the queries and
 * falls back (simple_tip_b200/core/stable_kde.py).  Same outputs as tip_kde_lse; pitch = tip_pair_pitch(d, 1). */
int tip_kde_lse_f16(const void* q_pack, int64_t m, const void* t_pack, int64_t n, int64_t d,
                    int64_t pitch, const tip_work_item* items, int32_t n_items, float* part_max,
                    float* part_sum, void* stream);
/* fp16 operand packing for tip_kde_lse_f16: row = [ h(fl32(x - center)) | tail ], tail(query) = [S,S,S,0..],
 * tail(train) = 3-way fp16 split of norm_coef*|v|^2/S with S = norm_scale (a power of two; keeps the norm
 * term in fp16's range).  sqnorm[rows] = |v|^2 (fp32, may be NULL); flags[0] |= 1 if anything left fp16's finite
 * range (flags may be NULL). */
int tip_pair_prep_f16(const void* src, int dtype, int64_t rows, int64_t d, const float* center, int role,
                      float norm_coef, float norm_scale, void* dst_f16, float* sqnorm, int32_t* flags,
                      void* stream);
/* merges `slots` partials per row into out_max, out_sum (fp32), in two levels: slot s goes to group s mod 8; each of
 * the 8 groups merges its slots online in ascending slot order (a higher max rescales the group's sum by
 * expf(old - new), a lower one adds part_sum * expf(part_max - max)); then the groups are merged in ascending group
 * order: out_max = the largest group max, out_sum = sum of group sum * expf(group max - out_max).  Slots whose
 * part_max is -inf (or NaN) are skipped; a row without any other slot gets (-inf, 0). */
int tip_kde_combine(const float* part_max, const float* part_sum, int64_t m, int32_t slots,
                    float* out_max, float* out_sum, void* stream);

/* ---- k-means discriminator of MultiModalSA (surprise.py:102-133) ---------------------------------
 * tip_kmeans_fit: x n x d (TIP_F32/TIP_F64, k <= n < 2^31), 1 <= k <= 64, 1 <= runs <= 64,
 * runs * k * d < 2^31, max_iter >= 0, tol >= 0.  Runs `runs` independent fits (sklearn's n_init) in one persistent cooperative
 * kernel.  Seeding: greedy k-means++ with 2 + int(ln k) trials per centre (first centre uniform,
 * candidates drawn with probability ~ D^2, the candidate with the lowest potential is kept); draws
 * come from a counter-based RNG keyed by (seed, k, run, step, trial).  Lloyd: nearest centre (squared
 * Euclidean in the input dtype, ties: lowest index), centres = member means accumulated in double.
 * Empty clusters (sklearn _relocate_empty_clusters): the set of empty clusters is fixed before any
 * row moves; in ascending cluster order each takes the row farthest from its centre (descending
 * distance, ties: lowest row), so a donor emptied by a move stays empty until the next assignment;
 * nothing moves when every row sits exactly on its centre (more clusters than distinct rows); a
 * cluster still empty keeps its previous centre.  A run stops when no label changed, when
 * sum ||centre shift||^2 <= tol (tol already scaled by the caller: mean(var(x, axis=0)) * tol), or
 * after max_iter iterations.  max_iter = 0 runs the seeding alone (centers = the seeds, n_iter = 0).
 * Writes centers[runs x k x d] (input dtype) and n_iter[runs]; the final labels / inertia come from
 * tip_kmeans_predict.  Deterministic:
 * fixed-order reductions, no floating-point atomics.  work: tip_kmeans_work_bytes(...) bytes of
 * scratch (-1: invalid arguments).  One call at a time per work buffer. */
int64_t tip_kmeans_work_bytes(int64_t n, int64_t d, int32_t k, int32_t runs, int dtype);
int tip_kmeans_fit(const void* x, int dtype, int64_t n, int64_t d, int32_t k, int32_t runs,
                   int32_t max_iter, double tol, uint64_t seed, void* work, void* centers,
                   int32_t* n_iter, void* stream);
/* labels[r*n + i] = nearest of the k centres centers[r] (runs x k x d, input dtype) to row i (ties:
 * lowest index); optional sqdist[r*n + i] (double) = its squared distance in the input dtype;
 * optional inertia[r] = sum_i sqdist[r*n + i] (double, fixed order; needs sqdist). */
int tip_kmeans_predict(const void* x, int dtype, int64_t n, int64_t d, const void* centers, int32_t k,
                       int32_t runs, int32_t* labels, double* sqdist, double* inertia, void* stream);

/* ---- silhouette score (sklearn.metrics.silhouette_samples) on the tensor cores ----------------------
 * tip_sil_prep: the rows src_idx[r] (label-sorted order; NULL: r) of x, centred on `center`, packed as
 * tip_pair_prep's three-segment operands — query role into q_pack, train role (scale -2, norm_coef 1)
 * into t_pack, pitch tip_pair_pitch(d, 3) — except that the norm term is the one the operands carry,
 * |h|^2 + 2<h, l>, so that identical rows give a distance of 0; sqnorm[rows] receives that norm.
 * tip_sil_dsum: for every work item (a query tile x a span of columns inside ONE cluster) writes
 * part_sum[slot*n + row] = sum over the span of sqrt(max(|x|^2 + |y|^2 - 2<x, y>, 0)), fp32, the row's
 * own column excluded (queries and columns are the same sorted matrix).
 * tip_sil_finish: out[out_idx[i]] (out_idx NULL: i) = silhouette value of sorted row i (double):
 * per-cluster sums merged over the slots in ascending order (slot_cluster[slots], non-decreasing),
 * a = sum_own / (n_own - 1), b = min over the other clusters of sum_c / n_c, (b - a) / max(a, b);
 * 0 for singleton clusters and for a = b = 0.  labels_sorted[n], counts[clusters]. */
int tip_sil_prep(const void* src, int dtype, int64_t rows, int64_t d, const float* center,
                 const int32_t* src_idx, void* q_pack, void* t_pack, float* sqnorm, void* stream);
int tip_sil_dsum(const void* q_pack, const void* t_pack, const float* sqnorm, int64_t n, int64_t d,
                 int64_t pitch, const tip_work_item* items, int32_t n_items, float* part_sum,
                 void* stream);
int tip_sil_finish(const float* part_sum, int64_t n, int32_t slots, const int32_t* slot_cluster,
                   const int32_t* labels_sorted, const int32_t* counts, const int32_t* out_idx,
                   double* out, void* stream);

/* ---- Gaussian mixture EM (sklearn GaussianMixture, covariance_type="full"), float64 ------------------
 * x n x d (TIP_F32/TIP_F64, widened exactly to double on load), 1 <= n < 2^31, 1 <= d <= 65536,
 * 1 <= k <= 64.  Parameters are double: means[k x d], prec_chol[k x d x d] (upper triangular, sklearn's
 * precisions_cholesky_; entries below the diagonal are never read), q / resp [k x n] (component-major).
 * Deterministic: fixed-order reductions, no floating-point atomics; the work split depends on the shape only.
 * tip_gmm_quad: q[j*n + i] = |(x_i - means_j) . prec_chol_j|^2 (centred first), fp64 tensor cores.
 * tip_gmm_resp: per row a_j = (-(d log 2pi + q_j) / 2 + log_det[j]) + log_weights[j]; optional
 *   lse[i] = logsumexp_j a_j (scipy order), labels[i] = first argmax_j a_j, resp[j*n + i] = exp(a_j - lse);
 *   optional lower_bound (device double) = mean of lse, merged in a fixed order (needs work).
 * tip_gmm_moments: nk[k] = sum_i resp + 10 eps(double), sums[k x d] = resp^T x, means = sums / nk; any
 *   of the three outputs may be NULL.
 * tip_gmm_scatter: S_j = sum_i resp[j*n+i] (x_i - means_j)(x_i - means_j)^T over lower-triangle tiles,
 *   mirrored; out[k x d x d] = S (nk NULL) or S / nk[j] + reg_covar on the diagonal.  The rows are split
 *   into tip_gmm_scatter_chunks(n, d, k, scatter_chunks) chunks (scatter_chunks 0: automatic; the count
 *   shrinks until the partials fit 256 MB) merged in ascending order.
 * work: tip_gmm_work_bytes(n, d, k, scatter_chunks) bytes, for any of the calls (-1: invalid). */
int32_t tip_gmm_scatter_chunks(int64_t n, int64_t d, int32_t k, int32_t scatter_chunks);
int64_t tip_gmm_work_bytes(int64_t n, int64_t d, int32_t k, int32_t scatter_chunks);
int tip_gmm_quad(const void* x, int dtype, int64_t n, int64_t d, const double* means,
                 const double* prec_chol, int32_t k, double* q, void* stream);
int tip_gmm_resp(const double* q, int64_t n, int64_t d, int32_t k, const double* log_weights,
                 const double* log_det, double* resp, double* lse, int64_t* labels, double* lower_bound,
                 void* work, void* stream);
int tip_gmm_moments(const void* x, int dtype, int64_t n, int64_t d, const double* resp, int32_t k,
                    double* nk, double* sums, double* means, void* work, void* stream);
int tip_gmm_scatter(const void* x, int dtype, int64_t n, int64_t d, const double* resp,
                    const double* means, int32_t k, const double* nk, double reg_covar,
                    int32_t scatter_chunks, double* out, void* work, void* stream);

/* ---- empirical covariance (sklearn EmpiricalCovariance.fit) --------------------------------------------
 * tip_cov_location: x n x d (TIP_F32/TIP_F64), 1 <= n < 2^31, 1 <= d <= 65536.  location[d] (x's dtype) =
 * X.mean(0) bit for bit as NumPy computes it (d >= 2: sequential sum over the rows in x's dtype; d == 1:
 * NumPy's pairwise sum), divided by n once; mean[d] (double) = the same sum in float64 / n, np.cov's centring
 * mean.  *flags (device int32, written by the call) = bit 0: some entry is NaN, bit 1: some entry is +-inf.
 * The scatter of the fit is tip_gmm_scatter with k = 1, unit weights, means = mean and nk = {n}. */
int tip_cov_location(const void* x, int dtype, int64_t n, int64_t d, void* location, double* mean,
                     int32_t* flags, void* stream);

/* ---- LSA's KDE fit (StableGaussianKDE on the device) ------------------------------------------------------
 * tip_col_var: x n x d (TIP_F32/TIP_F64), 1 <= n < 2^31, 1 <= d <= 65536.  var[d] (x's dtype) = np.var(x, axis=0)
 * bit for bit as NumPy 2.3's _methods._var computes it: the mean of tip_cov_location, then (x - mean) in x's
 * dtype, squared as a separate rounding, reduced like the mean (sequential over the rows for d >= 2, pairwise for
 * d == 1) and divided by n in double, rounded once.  mean[d] and *flags as tip_cov_location.
 * tip_whiten_dmma: out[m x d_out] (fp32) = (x[:, cols] - mu) . w, x: m x d_in (TIP_F32/TIP_F64), cols[d_out]
 * (NULL = all, then d_in == d_out), mu: d_out doubles, w: d_out x d_out doubles row-major, LOWER triangular
 * (entries above the diagonal are never read), 1 <= d_out <= 65536.  Accumulated in float64 on the fp64 tensor
 * cores, rounded once to fp32.  Deterministic (fixed order, no atomics). */
int tip_col_var(const void* x, int dtype, int64_t n, int64_t d, void* var, double* mean, int32_t* flags,
                void* stream);
int tip_whiten_dmma(const void* x, int dtype, int64_t m, int64_t d_in, const int32_t* cols, int64_t d_out,
                    const double* mu, const double* w_lower, float* out, void* stream);

/* ---- IMDB-C's dictionary distances (TextCorruptor) -------------------------------------------------------
 * tip_levenshtein: out[na x nb] (uint8, row-major, int64 indexing) = unit-cost Levenshtein distance (insert, delete,
 * substitute) of word a_i and word b_j, as polyleven.levenshtein computes it on Python str.  A word is a run of int32
 * code-point ids (equal ids = equal code points): a_ids[a_off[i] .. a_off[i+1]), a_off has na + 1 entries, likewise
 * b.  Ids below 64 get a shared-memory match mask, so the caller numbers the most frequent code points first; any
 * id >= 0 is exact.  max_len >= the longest word of a and b, <= 255 (so every distance fits in a byte).
 * symmetric != 0: a and b are the same block (same pointers, na == nb); each unordered pair is computed once and
 * written to both halves.  na == 0 or nb == 0 launches nothing. */
int tip_levenshtein(const int32_t* a_ids, const int32_t* a_off, int64_t na, const int32_t* b_ids,
                    const int32_t* b_off, int64_t nb, int32_t max_len, int symmetric, uint8_t* out, void* stream);

/* ---- the IMDB case study's inputs: Keras' word tokenizer (keras_preprocessing 1.1.2) -------------------------
 * Texts are one UTF-8 byte buffer text[text_off[t] .. text_off[t+1]) per text (n_texts + 1 offsets).  A word is a
 * maximal run of bytes that are not separators; separators are ASCII bytes, bit b of (sep_hi:sep_lo) set = byte b
 * separates (the filters and the split character).  Words are numbered text-major, position-minor.
 * tip_tok_count: lower != 0 lowercases ASCII A-Z in place; word_off[n_texts + 1] = exclusive scan of the words per
 * text (word_off[n_texts] = the total).
 * tip_tok_emit: w_start (byte offset), w_len, w_text and w_hash (64-bit hash of the bytes, low hash_bits bits
 * kept, 1..64; 64 in normal use, fewer only to force collisions) of every word; word_off from tip_tok_count.
 * tip_tok_vocab_table: the vocabulary (distinct words arena[v_start[i] .. + v_len[i])) into an open-addressing
 * table keys[cap] (cap a power of two >= 2 nv, <= 2^31; key = entry i, empty = ~0); v_hash[nv] out; first
 * (nullable) [cap] = the key of each slot, ~0 when empty (the fit's first-occurrence array).
 * tip_tok_fit: adds the n_words words to a table built by tip_tok_vocab_table with cap >= 2 (nv + n_words) and
 * first != nullptr.  A new word claims a slot with key nv + its first ordinal; words are compared by hash, length
 * and bytes, so collisions never merge words.  count / docs [cap] scratch, doc_keys [doc_cap] scratch (power of
 * two >= 2 n_words).  out [5][out_cap] (out_cap >= nv + n_words), one column per word this call saw, in no order:
 * first-occurrence key, occurrences, texts containing it, and for a new word (key >= nv) its first occurrence's
 * byte offset and length (else -1, 0); *n_out = the number of columns.
 * tip_tok_lookup: every word's id = v_index[its vocabulary entry] (keys from tip_tok_vocab_table), dropped when
 * unknown or when num_words != 0 and id >= num_words.  w_id [n_words] scratch; kept_off [n_texts + 1] = exclusive
 * scan of the kept ids per text; ragged (nullable, >= n_words entries) = the kept ids at kept_off; padded
 * (nullable) [n_texts][maxlen] = pad_sequences of the kept ids (maxlen >= 1, padding / truncating "pre" when
 * pre_padding / pre_truncating != 0, else "post", fill value).  n_texts == 0 launches nothing. */
int tip_tok_count(uint8_t* text, const int64_t* text_off, int64_t n_texts, uint64_t sep_lo, uint64_t sep_hi, int lower,
                  int64_t* word_off, void* stream);
int tip_tok_emit(const uint8_t* text, const int64_t* text_off, int64_t n_texts, uint64_t sep_lo, uint64_t sep_hi,
                 const int64_t* word_off, int64_t n_words, int32_t hash_bits, int64_t* w_start, int32_t* w_len,
                 int32_t* w_text, uint64_t* w_hash, void* stream);
int tip_tok_vocab_table(const uint8_t* arena, const int64_t* v_start, const int32_t* v_len, int64_t nv,
                        int32_t hash_bits, uint64_t* v_hash, uint64_t* keys, uint64_t* first, int64_t cap, void* stream);
int tip_tok_fit(const uint8_t* text, const int64_t* w_start, const int32_t* w_len, const int32_t* w_text,
                const uint64_t* w_hash, int64_t n_words, const uint8_t* arena, const int64_t* v_start,
                const int32_t* v_len, const uint64_t* v_hash, int64_t nv, uint64_t* keys, uint64_t* first,
                uint64_t* count, uint64_t* docs, int64_t cap, uint64_t* doc_keys, int64_t doc_cap, int64_t* out,
                int64_t out_cap, uint64_t* n_out, void* stream);
int tip_tok_lookup(const uint8_t* text, const int64_t* w_start, const int32_t* w_len, const uint64_t* w_hash,
                   int64_t n_words, const uint8_t* arena, const int64_t* v_start, const int32_t* v_len,
                   const uint64_t* v_hash, const int32_t* v_index, int64_t nv, const uint64_t* keys, int64_t cap,
                   int64_t num_words, const int64_t* word_off, int64_t n_texts, int32_t* w_id, int64_t* kept_off,
                   int32_t* ragged, int32_t* padded, int64_t maxlen, int pre_padding, int pre_truncating,
                   int32_t value, void* stream);

/* ---- IMDB-C's corruptions (TextCorruptor.corrupt) ----------------------------------------------------------
 * Texts are one strict UTF-8 byte buffer text[text_off[t] .. text_off[t+1]) per text (n_texts + 1 offsets,
 * n_texts < 2^31).  Every output is string for string what the host port's corrupt() returns.  The arithmetic:
 *   classes   cls[cp] for every code point present (TIP_CORRUPT_CP_WORDS * 32 entries): 0 whitespace (re's \s),
 *             1 word (re's \w), 2 other.  A word is a maximal run of class 1, or of class 2, code points
 *             (re.findall(r"\w+|[^\w\s]+", text)); words are numbered text-major, position-minor.
 *   md5mod(m) int(md5(m).hexdigest(), 16) % 10**6: the digest as a big-endian 128-bit integer.
 *   seeds     sentence seed S = md5mod(the text's words joined by single spaces) + seed (seed >= 0, S < 2^63);
 *             word i's seed s_i = S + i.
 *   rng(x)    NumPy's default_rng(x): SeedSequence(x).generate_state(4, uint64) = w0..w3 (x >= 2^32 enters as two
 *             little-endian uint32 words), PCG64 with inc = (w2:w3) << 1 | 1, state = 0, one step, state += w0:w1,
 *             one step; a step is state = state * 0x2360ED051FC65DA4_4385DF649FCCF645 + inc (mod 2^128); next64 =
 *             one step, then (hi ^ lo) rotated right by state >> 122; random() = (next64 >> 11) * 2^-53; uint32
 *             draws are buffered (one next64 gives its low half, then its high half).
 *   types     rng(S): one random() u per word, type = the entries of type_cdf[4] <= u (searchsorted, side right),
 *             type k being CorruptionType(k): 0 TYPO, 1 SYNONYM, 2 AUTOCOMPLETE, 3 AUTOCORRECT.
 *   chosen    a second rng(S) shuffles 0..n-1 as Generator.shuffle: for i = n-1 .. 1, swap i with j =
 *             random_interval(i) (mask = the smallest 2^b - 1 >= i, uint32 draws & mask until <= i); the first
 *             rint(n * severity) (half to even, in double) shuffled indexes are chosen.
 *   a chosen word w of >= 2 code points becomes, by its type (h = md5mod(w + " " + str(s_i))):
 *     TYPO          code point k = s_i % len(w) replaced by letter h % L of a..z without w[k] (L = 25 when w[k] is
 *                   in a..z, else 26);
 *     AUTOCOMPLETE  the values of the bag keyed by w's first min(5, len) code points, then 4, then 3, without w
 *                   itself: value h % (their number), in order; no such bag left: AUTOCORRECT;
 *     AUTOCORRECT   w unchanged unless it is a common-word key; then value v0 + (the entries of val_cdf[v0 .. v1) <=
 *                   rng(s_i).random()) of its range [v0, v1); an empty range sets *error_word = min(its word index)
 *                   (the host port's Generator.choice raises there);
 *     SYNONYM       the thesaurus value md5mod(w + " " + str(s_i) + " _corrupt_synonym") % (v1 - v0); no key or an
 *                   empty range: TYPO.
 *   output    each text's words (changed or not) joined by single spaces.
 * A table maps distinct keys (arena[key_off[i] .. + key_len[i]), n < 2^31) to value ranges val_begin[i] ..
 * val_begin[i+1] of strings arena[val_off[v] .. + val_len[v]); slots [cap] (cap a power of two >= 2 n) and key_hash
 * [n] are filled by tip_corrupt_table_build.  Lookups compare hash, length and bytes, so a hash collision never
 * changes a result.  val_cdf (common words only): Generator.choice's cdf of each key's candidates. */
#define TIP_CORRUPT_CP_WORDS 34816 /* 0x110000 / 32 */
typedef struct tip_corrupt_table {
  const uint8_t* arena;
  const int64_t* key_off;
  const int32_t* key_len;
  uint64_t* key_hash;
  const int64_t* val_begin;    /* [n + 1] */
  const int64_t* val_off;
  const int32_t* val_len;
  const double* val_cdf;       /* nullable except for the common-word table */
  int32_t* slots;              /* [cap], -1 = empty */
  int64_t n, cap;
} tip_corrupt_table;
/* tip_corrupt_table_build: key_hash and slots of a table (host struct, device arrays); n == 0 launches nothing.
 * tip_corrupt_census: bitmap [TIP_CORRUPT_CP_WORDS] = bit cp set for every non-ASCII code point of text[0, n_bytes).
 * tip_corrupt_count: n_words[t] = the words of text t.
 * tip_corrupt_texts: word_off [n_texts + 1] = exclusive scan of n_words; per word: w_start (byte offset), w_len
 *   (bytes), w_cps (code points), w_text, w_seed (s_i) and w_flags (type | 4 when chosen); perm [n_words] scratch.
 *   type_cdf is a HOST array of 4 doubles.
 * tip_corrupt_words: per word the result's source (o_src: 0 text, 1 common, 2 bags, 3 thesaurus arena), byte
 *   offset in it and length, and o_typo = -1 or (byte offset of the replaced code point << 16 | its byte length << 8
 *   | the letter); *error_word = 0x7f7f7f7f7f7f7f7f when no word failed.
 * tip_corrupt_layout: o_pos = each word's output offset within its text, text_len[t] = its output bytes.
 * tip_corrupt_write: out[out_off[t] + ...] = the output of text t (out_off: exclusive scan of text_len). */
int tip_corrupt_table_build(const tip_corrupt_table* table, void* stream);
int tip_corrupt_census(const uint8_t* text, int64_t n_bytes, uint32_t* bitmap, void* stream);
int tip_corrupt_count(const uint8_t* text, const int64_t* text_off, int64_t n_texts, const uint8_t* cls,
                      int64_t* n_words, void* stream);
int tip_corrupt_texts(const uint8_t* text, const int64_t* text_off, int64_t n_texts, const uint8_t* cls,
                      const int64_t* word_off, int64_t seed, double severity, const double* type_cdf, int64_t* w_start,
                      int32_t* w_len, int32_t* w_cps, int32_t* w_text, int64_t* w_seed, uint8_t* w_flags, int32_t* perm,
                      void* stream);
int tip_corrupt_words(const uint8_t* text, const int64_t* w_start, const int32_t* w_len, const int32_t* w_cps,
                      const int64_t* w_seed, const uint8_t* w_flags, int64_t n_words, const tip_corrupt_table* common,
                      const tip_corrupt_table* bags, const tip_corrupt_table* thesaurus, uint8_t* o_src, int64_t* o_off,
                      int32_t* o_len, int64_t* o_typo, int64_t* error_word, void* stream);
int tip_corrupt_layout(const int64_t* word_off, int64_t n_texts, const int32_t* o_len, const int64_t* o_typo,
                       int64_t* o_pos, int64_t* text_len, void* stream);
int tip_corrupt_write(const uint8_t* text, const int32_t* w_text, const int64_t* word_off, int64_t n_words,
                      const tip_corrupt_table* common, const tip_corrupt_table* bags,
                      const tip_corrupt_table* thesaurus, const uint8_t* o_src, const int64_t* o_off,
                      const int32_t* o_len, const int64_t* o_typo, const int64_t* o_pos, const int64_t* out_off,
                      uint8_t* out, void* stream);

/* ---- one training step of the case studies' models (case_study_*.py `model.fit`) -------------------------------
 * One parameter tensor of tip_keras_adam's table: param, its gradient and Adam's two moments, numel float32
 * elements each, all four laid out alike (element i of one is element i of the others). */
typedef struct tip_adam_tensor {
  float* param;
  const float* grad;
  float* m;
  float* v;
  int64_t numel;
} tip_adam_tensor;

/* tip_keras_adam: Keras' Adam (TF 2.6 optimizer_v2, amsgrad off, the "epsilon hat" form) over the n_tensors
 * (1..256) tensors of the DEVICE table, in one launch.  state[2] (device int32): state[0] = steps taken so far,
 * state[1] = 0 between calls (the kernel's arrival counter).  The step is t = state[0] + 1, and the kernel stores
 * state[0] = t, so a captured graph replays step after step.  Float32 operation order, each operation rounded
 * once (no FMA contraction):
 *   b1t = fl32(beta1 ^ t), b2t = fl32(beta2 ^ t)                (the powers in float64, rounded once)
 *   lr_t = lr * (sqrt(1 - b2t) / (1 - b1t))
 *   m = (beta1 * m) + ((1 - beta1) * g)
 *   v = (beta2 * v) + ((1 - beta2) * (g * g))
 *   param = param - ((lr_t * m) / (sqrt(v) + epsilon))
 * total_numel (the table's element count) only sizes the grid; a tensor's elements are read and written by one
 * thread each, with 16-byte accesses where its four arrays share their alignment.
 * tip_softmax_xent: the loss head of a step on logits z [rows x classes] (classes 1..32) and targets y (same
 * shape, float32): *loss = mean over rows of -sum_c y_c log softmax(z)_c, dz (nullable) = (softmax(z) - y) / rows,
 * *correct = rows whose first argmax of z equals the first argmax of y.  Fixed reduction order: the result
 * depends on the inputs only. */
int tip_keras_adam(const tip_adam_tensor* table, int32_t n_tensors, int64_t total_numel, int32_t* state, float lr,
                   float beta1, float beta2, float epsilon, void* stream);
int tip_softmax_xent(const float* z, const float* y, int64_t rows, int32_t classes, float* loss, float* dz,
                     int32_t* correct, void* stream);
/* tip_softmax_xent_seg: tip_softmax_xent on each of `segments` consecutive segments of rows_per_segment rows:
 * segment s (rows [s * rows_per_segment, (s + 1) * rows_per_segment) of z, y and dz) gives loss[s], its dz rows
 * divided by rows_per_segment and correct[s], bit for bit what tip_softmax_xent gives on that segment alone.
 * tip_softmax_xent is the launch with one segment. */
int tip_softmax_xent_seg(const float* z, const float* y, int64_t segments, int64_t rows_per_segment, int32_t classes,
                         float* loss, float* dz, int32_t* correct, void* stream);
/* tip_stack_gather: the batch of one step for `models` models trained in one stack.  pool [*, row_elems] (dtype
 * TIP_F32, TIP_F64 or TIP_I32, contiguous rows); rows [models][n_rows] (int64) = each model's pool rows; perm
 * [models][n_perm] (int64, values < n_perm <= n_rows) = each model's permutation of its first n_perm rows.  Row j
 * (j < b) of model m is pool row rows[m][perm[m][start + j]].  channels == 0: out [models][b][row_elems]
 * (model-major); channels > 0: out [b][P][models][channels] with P = row_elems / channels (an NHWC batch of
 * models * channels channels).  out is float32 for TIP_F32 and TIP_F64 (rounded to nearest), int32 for TIP_I32.
 * The pool row indexes are not range-checked here: the caller checks the rows table once. */
int tip_stack_gather(const void* pool, int32_t dtype, int64_t row_elems, const int64_t* rows, int64_t n_rows,
                     const int64_t* perm, int64_t n_perm, int64_t start, int64_t b, int64_t models, int64_t channels,
                     void* out, void* stream);

/* ---- MC-dropout head: the samples of a model's top-level dropout / dense chain ---------------------------
 * One layer of the head: a dropout of rate p on its input (p = 0: none), then the dense layer
 * y = act(x K + b) with K [in][out] (Keras' layout) and b [out], float32, contiguous, on the device. */
typedef enum tip_mc_activation { TIP_MC_LINEAR = 0, TIP_MC_RELU = 1, TIP_MC_SOFTMAX = 2 } tip_mc_activation;
typedef enum tip_mc_mode { TIP_MC_OUTPUT = 0, TIP_MC_PREACT = 1 } tip_mc_mode;
typedef struct tip_mc_layer {
  const float* kernel;     /* [in][out] */
  const float* bias;       /* [out] */
  double p;                /* dropout rate on the layer's input, 0 <= p <= 1 */
  int32_t in, out;         /* layer 0: 1 <= in <= 8192; later layers: in = the previous out; 1 <= out <= 64 */
  int32_t activation;      /* tip_mc_activation; TIP_MC_SOFTMAX only on the last layer */
  int32_t reserved;        /* 0 */
} tip_mc_layer;
/* tip_mc_head: h [rows][ld] float32 (the first `in` columns of each row are the trunk activations; row i is the
 * global row row0 + i); layers [n_layers] (1..4, host memory).  For every row i < rows and sample s < samples,
 * out[(i * samples + s) * C + c] (C = the last layer's out) receives the last layer's output (mode TIP_MC_OUTPUT)
 * or its pre-activation x K + b (TIP_MC_PREACT, for tests) for the global sample sample0 + s.
 *
 * Arithmetic (restatable bit for bit):
 *   key(l, r, s) = mix(mix(mix(mix(seed) ^ l) ^ r) ^ s), mix = one splitmix64 step, l = the layer's index in
 *     `layers`, r = row0 + i, s = sample0 + s;
 *   u(l, r, s, j) = the low (j even) or high (j odd) 32 bits of mix(key(l, r, s) ^ (j >> 1)) for input unit j;
 *   unit j is dropped iff u < t, t = rint(p * 2^32) (p = 1 drops every unit);
 *   x'_j = 0 if dropped, else x_j * scale rounded once, scale = float32(1 / float32(1 - p)) (torch's dropout);
 *   z_c = ((...((0 + x'_0 K[0][c]) + x'_1 K[1][c]) + ...) + x'_{in-1} K[in-1][c]) + b[c], every product and sum
 *     rounded once to float32 (no FMA), units in ascending order;
 *   relu: z < 0 ? 0 : z (NaN stays NaN); softmax: m = max_c z_c, e_c = expf(z_c - m), s = sum of e_c in class
 *     order, y_c = e_c / s.
 * The draws depend on (seed, l, r, s, j) only: not on the launch shape, the row split or the sample split. */
int tip_mc_head(const float* h, int64_t rows, int64_t ld, int64_t row0, int64_t sample0, int64_t samples,
                const tip_mc_layer* layers, int32_t n_layers, uint64_t seed, int32_t mode, float* out, void* stream);
/* tip_mc_head_stack: tip_mc_head on `models` heads of one shape (a stack's), in one launch per 256 models.
 * layers[l].kernel is [models][in][out] and layers[l].bias [models][out]; model m's row i of h starts at
 * h + m * ldm + i * ld (ldm = 0: every model reads the same rows); seeds [models] (host memory) = one seed per model;
 * out [models][rows][samples][C].  out[m] is bit for bit what tip_mc_head writes for model m's h, kernels, biases
 * and seeds[m] (same rows, row0, sample0, samples, rates, activations and mode): the key above with seed = seeds[m],
 * so the model index enters through the seed only. */
int tip_mc_head_stack(const float* h, int64_t models, int64_t rows, int64_t ld, int64_t ldm, int64_t row0,
                      int64_t sample0, int64_t samples, const tip_mc_layer* layers, int32_t n_layers,
                      const uint64_t* seeds, int32_t mode, float* out, void* stream);

/* ---- bring-up / validation: plain accumulator dump ------------------------------------
 * out[256*256] (fp32, row-major, leading dimension 256) = tail-augmented dot products of q rows
 * [0,128) with t rows [0,256).
 * variant: 0 = the kernel tip_nn_filter would pick, 1 = streaming, 2 = resident-query. */
int tip_pair_probe(const void* q_pack, int64_t m, const void* t_pack, int64_t n, int64_t d,
                   int segments, int64_t pitch, int variant, float* out, void* stream);

/* bring-up: while buf != NULL, block 0 of the filter kernel records clock64() stamps (16 int64 slots
 * per train tile, up to `tiles` tiles): 0 / 1 first consumer warp before the tile's first chunk wait /
 * after its last wgmma, 7 the same warp at the end of the tile's reduction, 8 / 10 TMA producer before /
 * after issuing the tile's loads. */
int tip_debug_timeline(long long* buf, int32_t tiles);
/* bring-up: while buf != NULL, every CTA of the filter kernel writes
 * {globaltimer ns at start, at end, train tiles, work items} to buf[4*blockIdx.x ...]. */
int tip_debug_cta_clock(long long* buf);

#ifdef __cplusplus
}
#endif
#endif /* B200TIP_H */
