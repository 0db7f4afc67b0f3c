/* mtadgat.h -- C ABI of libmtadgat.so, the H100 (sm_90a) hot path of MTAD-GAT.
 *
 * The reference (ML4ITS/mtad-gat-pytorch) has no FFI: its boundary for this path is the set of Python
 * nn.Module classes in modules.py / mtad_gat.py.  Each entry point below replaces the arithmetic of one of
 * those classes' forward (and the autograd backward torch derives for it); the citation after each
 * declaration is the reference file:line it stands in for.  The Python host side
 * (mtad_gat_pytorch_b200/modules.py) mirrors the reference classes and calls these through ctypes.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to contiguous fp32 unless stated otherwise; sizes are ints
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises
 *   - one device per process (the scaling model is one process per GPU): the mode switches (mtadgat_set_*), the per-stream
 *     pack workspaces and the kernels' one-time attribute setup are process-wide and assume the calling thread's current
 *     device is the one the pointers live on
 *   - return value 0 = ok; non-zero = error, message via mtadgat_last_error() (thread-local)
 *   - `saved` buffers are written by *_fwd and must be handed unchanged to the matching *_bwd;
 *     `scratch` buffers are temporaries; sizes (in floats) come from the *_floats() queries
 *   - dropout: multipliers are a pure function of (*seed, rng stream id, element index) (Philox4x32-10), so
 *     forward and backward regenerate the same mask; `seed` points to a device uint64 (CUDA-graph safe)
 *   - gradients of parameters are overwritten (not accumulated); data gradients honour `*_accumulate`
 *   - `parts` of a *_bwd: bit 0 = recurrence / data-gradient work (the critical path of backpropagation),
 *     bit 1 = parameter-gradient work (reads what bit 0 left in `scratch`).  3 = everything on `stream`;
 *     the host layer issues 1 on the main stream and 2 on a side stream so parameter gradients overlap the
 *     upstream layers' backward.  mtadgat_gat_bwd additionally takes 1|8 (score backward without the final dV products)
 *     and 4 (those products alone): issued as 1|8 (main), 2 (side), 4 (main), the parameter GEMMs start as soon as the
 *     score backward is done.
 */
#ifndef MTADGAT_H_
#define MTADGAT_H_

#ifdef __cplusplus
extern "C" {
#endif

#define MTADGAT_ABI_VERSION 3

const char* mtadgat_last_error(void);
int mtadgat_abi_version(void);
unsigned long long mtadgat_launch_count(void);     /* kernels launched by this library so far */
void mtadgat_reset_launch_count(void);

/* ---- ConvLayer.forward: modules.py:18-22 (pad, Conv1d, ReLU; x,y are (B,n,k); w (k,k,ks); odd ks) ---- */
int mtadgat_conv_relu_fwd(const float* x, const float* w, const float* bias, float* y, int B, int n, int k, int ks,
                          void* stream);
int mtadgat_conv_relu_bwd(const float* x, const float* w, const float* y, const float* dy, float* dx /*nullable*/,
                          float* dw, float* db, int B, int n, int k, int ks, void* stream);
/* same, for an output that feeds several consumers (mtad_gat.py:68-71: both GAT layers and the GRU read the conv
 * output): the consumers' gradients dy, dy1, dy2 (dy1 / dy2 nullable) are summed inside the kernels */
int mtadgat_conv_relu_bwd3(const float* x, const float* w, const float* y, const float* dy, const float* dy1,
                           const float* dy2, float* dx /*nullable*/, float* dw, float* db, int B, int n, int k, int ks,
                           void* stream);

/* ConvLayer over B windows that start x_window_stride ELEMENTS apart: stride k = the overlapping slices of a
 * device-resident (N,k) series (utils.py:107-120 SlidingWindowDataset.__getitem__, prediction.py:43-52), read in place. */
int mtadgat_conv_relu_fwd_strided(const float* x, const float* w, const float* bias, float* y, int B, int n, int k, int ks,
                                  long long x_window_stride, void* stream);

/* ---- FeatureAttentionLayer.forward modules.py:65-95 (feature=1) / TemporalAttentionLayer.forward
 *      modules.py:166-193 (feature=0).  E = lin.weight.shape[0]; GATv2: lin_w (E,2D), a (E); GATv1: lin_w (E,D),
 *      a (2E); D = n (feature) or k (temporal); bias (K,K) nullable; out (B,n,k).
 *      save_att=1 keeps the attention matrix in `saved` for backward; p_drop = attention dropout
 *      (0 in eval mode).  rng stream ids 1 (feature) and 2 (temporal) are used internally. ---- */
long long mtadgat_gat_saved_floats(int B, int n, int k, int E, int feature, int use_gatv2, int save_att);
long long mtadgat_gat_bwd_scratch_floats(int B, int n, int k, int E, int feature, int use_gatv2);
int mtadgat_gat_fwd(const float* x, const float* lin_w, const float* lin_b, const float* a, const float* bias,
                    float* out, float* saved, int B, int n, int k, int E, int feature, int use_gatv2, float alpha,
                    int save_att, float p_drop, const unsigned long long* seed, void* stream);
int mtadgat_gat_bwd(const float* x, const float* lin_w, const float* lin_b, const float* a, const float* out,
                    const float* gout, const float* saved, float* scratch, float* dx, int dx_accumulate,
                    float* dlin_w, float* dlin_b, float* da, float* dbias /*nullable*/, int B, int n, int k, int E,
                    int feature, int use_gatv2, float alpha, float p_drop, const unsigned long long* seed,
                    int parts, void* stream);

/* ---- GRULayer.forward modules.py:235-238 (one nn.GRU layer, batch_first, h0=0, gate order r,z,n).
 *      The input is given as up to three column slices x0|x1|x2 of widths k0,k1,k2 (the torch.cat of
 *      mtad_gat.py:71 is never materialised).  out (B,n,H) nullable when save=0; h_last (B,H) nullable. ---- */
long long mtadgat_gru_saved_floats(int B, int n, int H, int save);
long long mtadgat_gru_fwd_scratch_floats(int B, int n, int H);
long long mtadgat_gru_bwd_scratch_floats(int B, int n, int H);
int mtadgat_gru_fwd(const float* x0, const float* x1, const float* x2, int k0, int k1, int k2, const float* w_ih,
                    const float* w_hh, const float* b_ih, const float* b_hh, float* out, float* h_last, float* saved,
                    float* scratch, int B, int n, int H, int save, void* stream);
int mtadgat_gru_bwd(const float* x0, const float* x1, const float* x2, int k0, int k1, int k2, const float* w_ih,
                    const float* w_hh, const float* out, const float* saved, const float* dout /*nullable*/,
                    const float* dh_last /*nullable*/, float* scratch, float* dx0, float* dx1, float* dx2, int acc0,
                    int acc1, int acc2, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh, int B, int n, int H,
                    int parts, void* stream);

/* ---- ReconstructionModel.forward modules.py:276-281: decoder GRU over the reference's scrambled repeat
 *      rep[b,t,c] = h_src[b,(t*Hs+c)//n] (modules.py:279), all n outputs (B,n,R). ---- */
int mtadgat_rep_J(int n, int Hs);
long long mtadgat_gru_rep_saved_floats(int B, int n, int Hs, int R, int save);
long long mtadgat_gru_rep_bwd_scratch_floats(int B, int n, int Hs, int R);
int mtadgat_gru_rep_fwd(const float* h_src, const float* w_ih, const float* w_hh, const float* b_ih,
                        const float* b_hh, float* out, float* saved, int B, int n, int Hs, int R, int save,
                        void* stream);
int mtadgat_gru_rep_bwd(const float* h_src, const float* w_ih, const float* w_hh, const float* out,
                        const float* saved, const float* dout, float* scratch, float* dh_src, int dh_accumulate,
                        float* dw_ih, float* dw_hh, float* db_ih, float* db_hh, int B, int n, int Hs, int R,
                        int parts, void* stream);

/* Scoring path: the same decoder emitting only its last state h_{n-1} (B,R) (prediction.py:62 keeps
 * window_recon[:, -1, :] only).  scratch: mtadgat_gru_rep_saved_floats(B,n,Hs,R,0) floats. */
int mtadgat_gru_rep_last(const float* h_src, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                         float* h_last, float* scratch, int B, int n, int Hs, int R, void* stream);

/* ---- nn.Linear (+ReLU, +Dropout): Forecasting_Model.forward modules.py:307-311, recon fc modules.py:282.
 *      x (M,I), w (O,I), b (O), y (M,O); act 0 none / 1 relu. ---- */
int mtadgat_linear_fwd(const float* x, const float* w, const float* b, float* y, int M, int I, int O, int act,
                       float p_drop, const unsigned long long* seed, unsigned int rng_stream, void* stream);
int mtadgat_linear_bwd(const float* x, const float* w, const float* y, const float* dy, float* dx /*nullable*/,
                       int dx_accumulate, float* dw, float* db, float* scratch /* M*O floats; nullable if act=0,p=0 */,
                       int M, int I, int O, int act, float p_drop, const unsigned long long* seed,
                       unsigned int rng_stream, int parts, void* stream);

/* ---- the training loss of the reference step (training.py:113-124), both terms in one pass:
 *      losses[0] = sqrt(mean((y - preds)^2)) over n_pred elements, losses[1] = sqrt(mean((x - recons)^2)) over n_rec.
 *      sums: 2 doubles of scratch.  bwd: dpreds = g_forecast * (preds - y) / (n_pred * losses[0]) (same for recons);
 *      g_* are device scalars (the upstream gradients), dpreds / drecons nullable. ---- */
int mtadgat_rmse_pair_fwd(const float* preds, const float* y, long long n_pred, const float* recons, const float* x,
                          long long n_rec, float* losses, double* sums, void* stream);
int mtadgat_rmse_pair_bwd(const float* preds, const float* y, long long n_pred, const float* recons, const float* x,
                          long long n_rec, const float* losses, const float* g_forecast, const float* g_recon,
                          float* dpreds, float* drecons, void* stream);

/* ---- the optimiser step of the reference loop (train.py:92 torch.optim.Adam, training.py:127 optimizer.step()) over ALL
 *      parameter tensors in one launch: table = n_tensors x 5 device int64 {param, grad, exp_avg, exp_avg_sq, numel} (fp32
 *      tensors), step = device float holding the number of steps taken so far (incremented here; graph-replay safe).
 *      No weight decay, no amsgrad (the reference uses neither). ---- */
int mtadgat_adam_step(const long long* table, int n_tensors, long long max_numel, float lr, float beta1, float beta2,
                      float eps, float* step, void* stream);

/* ---- training epochs from a device-resident (N,k) series (training.SeriesTrainer).  `counter` is one device int64,
 *      the step of the epoch: both calls read it, so a captured CUDA graph replays a whole epoch with no host work.
 *      mtadgat_gather_windows: utils.py:107-120 SlidingWindowDataset.__getitem__ + the DataLoader's collate.  For
 *      b < count, with i = idx[*counter * ld + b] (idx: a (steps, ld) device int64 table of window starts, trusted:
 *      0 <= i <= N-n-1), x[b] = series[i : i+n] (n*k floats) and y[b] = series[i+n] (k floats); x (count,n,k),
 *      y (count,1,k).  count <= ld.  Does not change *counter.
 *      mtadgat_record_step: training.py:129-130 `forecast_b_losses.append(forecast_loss.item())` /
 *      `recon_b_losses.append(recon_loss.item())` (and the same lists of Trainer.evaluate): table[2 * *counter + j] =
 *      losses[j], j = 0, 1 (table: (steps, 2) device floats), then ++*counter. ---- */
int mtadgat_gather_windows(const float* series, const long long* idx, long long ld, const long long* counter, int count,
                           int n, int k, float* x, float* y, void* stream);
int mtadgat_record_step(const float* losses, float* table, long long* counter, void* stream);

/* ---- anomaly-score epilogue of Predictor.get_score (prediction.py:65-91): a_score[i][c] = |preds[i][c] - actual| +
 *      gamma |recons_last[i][c] - actual|, actual = series[n+i][target_dims ? target_dims[c] : c]; a_global[i] = mean_c
 *      (nullable).  preds, recons_last, a_score are (n_windows, out); series (N,k) with N >= n + n_windows;
 *      target_dims: `out` device ints or NULL. ---- */
int mtadgat_score_epilogue(const float* preds, const float* recons_last, const float* series, const int* target_dims,
                           int n, int k, int out, long long n_windows, float gamma, float* a_score,
                           float* a_global /*nullable*/, void* stream);

/* ---- epsilon threshold (Hundman et al.) on the anomaly scores, as eval_methods.py:186-236 find_epsilon computes it
 *      (19 candidates mean + z*sd, z = 2.5 .. 11.5; anomalies dilated by +-49 indices; reg_level 0/1/2).  scores: n_scores
 *      device floats (e.g. a_global of mtadgat_score_epilogue).  out[0] = epsilon, out[1] = the winning z (-1: no
 *      candidate qualified, epsilon = max(scores)), out[2] = its score.  scratch: mtadgat_find_epsilon_scratch_doubles(n_scores) doubles.
 *      All sums are formed in a fixed order (no floating-point atomics): candidates with the same pruned set tie exactly,
 *      and ties go to the last candidate as in the reference. ---- */
long long mtadgat_find_epsilon_scratch_doubles(long long n_scores);
int mtadgat_find_epsilon(const float* scores, long long n_scores, int reg_level, float* out, double* scratch, void* stream);
/* the same for each column of a row-strided (n_rows, n_cols) matrix in one launch sequence (prediction.py's per-feature
 * find_epsilon(A_Score_i, reg_level=2)): column c is x[i*ld + c].  Doubles out[c] = epsilon, out[n_cols + c] = z,
 * out[2*n_cols + c] = score.  A column's result is bitwise the same whatever matrix it is part of, and its float
 * rounding is what mtadgat_find_epsilon returns for it.  scratch: mtadgat_find_epsilon_columns_scratch_doubles doubles. */
long long mtadgat_find_epsilon_columns_scratch_doubles(long long n_rows, int n_cols);
int mtadgat_find_epsilon_columns(const float* x, long long n_rows, int n_cols, long long ld, int reg_level, double* out,
                                 double* scratch, void* stream);
/* the same on a row-strided float64 matrix (the float64 A_Score_i of scale_scores=True); the column arithmetic is the
 * float32 entry's, on the double values.  scratch: mtadgat_find_epsilon_columns_scratch_doubles doubles. */
int mtadgat_find_epsilon_columns_f64(const double* x, long long n_rows, int n_cols, long long ld, int reg_level,
                                     double* out, double* scratch, void* stream);

/* ---- point-adjusted evaluation of thresholds on the anomaly scores, eval_methods.py `adjust_predicts` +
 *      `calc_point2point` (run T times by `bf_search`, once by `epsilon_eval` and `pot_eval`).  actual = labels > 0.1; an
 *      anomaly segment is a maximal run of actual points; a segment with a raw prediction in it is predicted in full
 *      from its start (index 0 excepted: the reference's back-fill `range(i, 0, -1)` stops at 1) and adds the points it
 *      back-filled to the latency.  The raw prediction is `scores[i] > thr` (ge = 0) or `>= thr` (ge = 1), compared in
 *      double (a caller that wants numpy's float32 comparison rounds thr to float32 first), or, with `pred` (device uint8
 *      0/1, the reference's pred=) instead of `scores`, pred[i] itself.  Pass exactly one of scores / pred, the same
 *      one to every call on one `segs`.  Every count is an exact integer.
 *      1. mtadgat_eval_segments, once per (scores or pred, labels): segments, their running score maxima and the number
 *         of labels that are not exactly 0 or 1 into `segs` (mtadgat_eval_segments_words(n) int64 words; read by 2, 3).
 *      2. mtadgat_eval_counts: counts[6*t ..] = {TP, TN, FP, FN, latency_sum, n_detected} (int64) for thresholds[t]
 *         (n_thr device doubles; with pred: n_thr = 1, thresholds NULL).  All six are -1 when a label is not 0 / 1
 *         (calc_point2point weights by the raw label).  scratch: mtadgat_eval_counts_scratch_words(n, n_thr) int64.
 *         latency = latency_sum / (n_detected + 1e-4) as the reference returns it.
 *      3. mtadgat_eval_predict: the point-adjusted predictions for one threshold, out[i] = 0 / 1 (uint8, n).
 *      labels: n device floats; n < 2^31.  No allocation, no synchronisation (CUDA-graph capturable). ---- */
long long mtadgat_eval_segments_words(long long n);
int mtadgat_eval_segments(const float* scores /*nullable*/, const unsigned char* pred /*nullable*/, const float* labels,
                          long long n, long long* segs, void* stream);
long long mtadgat_eval_counts_scratch_words(long long n, int n_thr);
int mtadgat_eval_counts(const float* scores /*nullable*/, const unsigned char* pred /*nullable*/, long long n,
                        const long long* segs, const double* thresholds, int n_thr, int ge, long long* counts,
                        long long* scratch, void* stream);
int mtadgat_eval_predict(const float* scores /*nullable*/, const unsigned char* pred /*nullable*/, long long n,
                         const long long* segs, double threshold, int ge, unsigned char* out, void* stream);
/* mtadgat_eval_counts for n_rows prediction rows at once (thresholding.replay_eval): row r is pred[r*ld : r*ld + n]
 * (device uint8, ld >= n; any nonzero byte is a prediction, so biSPOT's codes 1 and 2 both count), all counted against
 * one `segs` of mtadgat_eval_segments on the labels (the running maxima in it are not read).  counts[6*r ..] as
 * mtadgat_eval_counts writes them for pred = row r alone, bitwise; integer per-block partials, one launch plus the
 * finishing one for all rows.  scratch: mtadgat_eval_counts_scratch_words(n, n_rows) int64.  n_rows <= 65535. */
int mtadgat_eval_counts_rows(const unsigned char* pred, long long n, int n_rows, long long ld, const long long* segs,
                             long long* counts, long long* scratch, void* stream);
/* PA%K, point adjustment only for segments with more than K % of their points predicted (Kim et al., AAAI 2022), on a
 * `segs` of mtadgat_eval_segments.  At threshold t (the raw prediction is scores[i] > t, compared in double) or for a
 * prediction row (nonzero byte = predicted), anomaly segment j of length L with d predicted points qualifies at K when
 * 100 * d > K * L (integers); a qualifying segment adds to TP what adjust_predicts gives a detected one, L, or L - 1
 * when it starts at index 0 and index 0 is not predicted; any other segment adds d.  FP = predicted normal points,
 * TN = N - FP, FN = P - TP.  K = 0 is adjust_predicts + calc_point2point exactly; K = 100 the point-wise confusion.
 * ks: n_k <= 101 strictly increasing integers in [0, 100] (HOST ints).  All four counts are -1 when a label is not 0 / 1.
 *      mtadgat_eval_pak_counts: counts[(k*n_thr + t)*4 ..] = {TP, TN, FP, FN} (int64) for K = ks[k] and thresholds[t]
 *      (n_thr device doubles, at most 65535 * 8).
 *      mtadgat_eval_pak_counts_rows: counts[(r*n_k + k)*4 ..] for row r = pred[r*ld : r*ld + n] (device uint8, ld >= n,
 *      n_rows <= 65535); at K = 0 bitwise mtadgat_eval_counts_rows' TP, TN, FP, FN.
 *      scratch: mtadgat_eval_pak_scratch_words(n, n_thr or n_rows, n_k) int64.  Integer per-block partials, one count
 *      launch and one finishing launch. */
long long mtadgat_eval_pak_scratch_words(long long n, int n_thr, int n_k);
int mtadgat_eval_pak_counts(const float* scores, long long n, const long long* segs, const double* thresholds, int n_thr,
                            const int* ks, int n_k, long long* counts, long long* scratch, void* stream);
int mtadgat_eval_pak_counts_rows(const unsigned char* pred, long long n, int n_rows, long long ld, const long long* segs,
                                 const int* ks, int n_k, long long* counts, long long* scratch, void* stream);
/* out[i*n_cols + c] = x[i*ld + c] > thresholds[c] (ge = 0) or >= (ge = 1), compared in double, as uint8 0 / 1:
 * prediction.py's per-feature A_Pred_i = (A_Score_i >= epsilon_i) for the epsilons of mtadgat_find_epsilon_columns. */
int mtadgat_compare_columns(const float* x, long long n, int n_cols, long long ld, const double* thresholds, int ge,
                            unsigned char* out, void* stream);
int mtadgat_compare_columns_f64(const double* x, long long n, int n_cols, long long ld, const double* thresholds, int ge,
                                unsigned char* out, void* stream);

/* ---- affiliation precision and recall (Huet, Navarro and Rossi, KDD 2022) of 0/1 predictions against the m anomaly
 *      events of a `segs` of mtadgat_eval_segments on the labels, n < 2^24.  Event j = [s_j, e_j) (e_j exclusive), zone
 *      I_j = [b_{j-1}, b_j) cut at the midpoints b_j = (e_j + s_{j+1}) / 2 (b = 0 before the first, n after the last);
 *      Y_j = the predicted units [i, i+1) within I_j.  Per (row, zone) three exact integers,
 *      words[(r*zone_cap + j)*3 ..] = {8 * integral over Y_j of |I_j| Fbar_j(dist(y, J_j)), 2 |Y_j|,
 *      16 * integral over J_j of |I_j| G_j(dist(x, Y_j))}, and
 *      probs[(2r)*zone_cap + j] = P_j = word0 / (8 |I_j| |Y_j|) (NaN when |Y_j| = 0),
 *      probs[(2r + 1)*zone_cap + j] = R_j = word2 / (16 |I_j| |J_j|), each one float64 division (every integer < 2^53).
 *      out (2 + 3 * rows int64): [0] m, [1] status (MTADGAT_AFF_*), then per row {mean of the defined P_j (NaN when none)
 *      and mean of all R_j as double bits, numpy's pairwise sum divided by the count (np.mean); the number of zones with
 *      |Y_j| > 0}.  zone_cap: the zone slots per row of words / probs, m <= zone_cap <= n / 2 + 1 (MTADGAT_AFF_CAPACITY
 *      and nothing per zone written when m > zone_cap).  rows <= 65535.  scratch:
 *      mtadgat_affiliation_scratch_words(n, rows, zone_cap) int64.  Integer atomics, no allocation, no synchronisation,
 *      six launches whatever n and rows; bitwise repeatable; safe with m = 0 (MTADGAT_AFF_NO_EVENT).
 *      mtadgat_affiliation_rows: row r = pred[r*ld : r*ld + n] (device uint8, nonzero = predicted, ld >= n).
 *      mtadgat_affiliation_thresholds: row t = scores > thresholds[t] (device float32 scores, n_thr device doubles,
 *      compared in double; NaN never predicted). ---- */
#define MTADGAT_AFF_NO_EVENT 1
#define MTADGAT_AFF_BAD_LABEL 2
#define MTADGAT_AFF_CAPACITY 4
long long mtadgat_affiliation_scratch_words(long long n, int n_rows, long long zone_cap);
int mtadgat_affiliation_rows(const unsigned char* pred, long long n, int n_rows, long long ld, const long long* segs,
                             long long zone_cap, long long* words, double* probs, long long* out, long long* scratch,
                             void* stream);
int mtadgat_affiliation_thresholds(const float* scores, long long n, const long long* segs, const double* thresholds,
                                   int n_thr, long long zone_cap, long long* words, double* probs, long long* out,
                                   long long* scratch, void* stream);

/* ---- threshold-free evaluation of anomaly scores: ROC-AUC and average precision (sklearn's roc_auc_score and
 *      average_precision_score) of n device floats `scores` against n device float `labels` (1 positive, 0 negative),
 *      n < 2^27.  Ties are IEEE equality (-0.0 == +0.0).
 *      ROC-AUC = U / (2 * P * N) in one float64 division, U = sum over positives of (2 * #negatives below + #negatives
 *      tied), an exact integer: the correctly rounded tie-averaged AUC; NaN when P or N is 0.
 *      AP: over each distinct positive score v in descending order, with tps / fps the positives / negatives >= v, the
 *      term (tps(v) - tps(previous v)) / P * (tps(v) / (tps(v) + fps(v))) (three float64 operations), the terms summed
 *      in that order by numpy's pairwise sum (np.sum); 0.0 when P = 0, 1.0 when N = 0.
 *      out (5 int64 words): [0] ROC-AUC and [1] AP as double bits, [2] P, [3] N, [4] status: MTADGAT_AUC_NONFINITE (a
 *      NaN or infinite score), MTADGAT_AUC_BAD_LABEL (a label other than 0 / 1; the results are then meaningless).
 *      scratch: mtadgat_auc_scratch_words(n) int64.  The scores are split by class, each class sorted by a keys-only
 *      LSD radix sort; 19 launches whatever n, no allocation, no synchronisation, no floating-point atomics, bitwise
 *      repeatable. ---- */
#define MTADGAT_AUC_NONFINITE 1
#define MTADGAT_AUC_BAD_LABEL 2
long long mtadgat_auc_scratch_words(long long n);
int mtadgat_auc(const float* scores, const float* labels, long long n, long long* out, long long* scratch, void* stream);

/* ---- anomaly diagnosis: the features of each timestamp ranked by score, and OmniAnomaly's HitRate@P% / NDCG@P% of the
 *      ranking against per-feature labels, as TranAD's diagnosis.py `hit_att` / `ndcg` compute them.  a: the row-strided
 *      (m, out) device float32 / float64 score matrix (row i is a[i*ld .. i*ld + out), ld >= out), read in place;
 *      2 <= out <= 1024, m < 2^31 - 1.
 *      mtadgat_rank_features: order (m, out) device int32, order[i*out + r] = the feature at rank r of row i, exactly
 *      np.argsort(-a[i], kind="stable"): descending score, ties (IEEE equality, -0.0 == +0.0) to the lower feature index,
 *      NaN last in index order, infinities ordinary values.  One launch.
 *      mtadgat_diagnose: labels (m, out) device uint8 0 / 1 with row stride ld_labels >= out; rows: n_masks row masks
 *      (n_masks, m) device uint8, any nonzero byte selecting the row (biSPOT's alarm code 2 too), or NULL for every row
 *      with n_masks = 1 (n_masks <= 65535); ps: n_p <= 16 cutoff percentages P, finite and >= 100 (HOST doubles).
 *      Per row i with g > 0 labelled features (label 1; rows with g = 0 are skipped, as TranAD skips them): cutoff
 *      k = min(rint((P * g) / 100.0), out) (Python's round(p * len(l) / 100)); Hit = (labelled features among the first
 *      k of the ranking above) / g in double; NDCG = sklearn's ndcg_score(l, a, k=k) with ignore_ties=False: the tie-averaged DCG (each tie
 *      group's mean gain times the sum of its positions' discounts 1 / log2(pos + 2), discounts at pos >= k zero) over
 *      IDCG = sum_{j < min(g, k)} 1 / log2(j + 2).  means[(r*n_p + p)*2 + {0, 1}] (doubles) = the mean Hit / NDCG at
 *      ps[p] over the rows mask r selects that have g > 0: numpy's pairwise float64 sum of the per-row values in row
 *      order, / their count (np.mean of the list; NaN for no row); counts[r] (int64) = that count; *status (int64) = bit
 *      0 a NaN score in an evaluated row, bit 1 a label other than 0 / 1 anywhere.  scratch:
 *      mtadgat_diagnose_scratch_words(m, n_masks, n_p) int64 words (4 * n_masks * m bytes of it a row index per mask).
 *      Three launches whatever m, n_masks and n_p.
 *      Both: no allocation, no synchronisation, no floating-point atomics, fixed reduction orders (bitwise repeatable;
 *      CUDA-graph capturable). ---- */
int mtadgat_rank_features(const float* a, long long m, int out, long long ld, int* order, void* stream);
int mtadgat_rank_features_f64(const double* a, long long m, int out, long long ld, int* order, void* stream);
long long mtadgat_diagnose_scratch_words(long long m, int n_masks, int n_p);
int mtadgat_diagnose(const float* a, long long m, int out, long long ld, const unsigned char* labels, long long ld_labels,
                     const unsigned char* rows /*nullable*/, int n_masks, const double* ps, int n_p, double* means,
                     long long* counts, long long* status, long long* scratch, void* stream);
int mtadgat_diagnose_f64(const double* a, long long m, int out, long long ld, const unsigned char* labels,
                         long long ld_labels, const unsigned char* rows /*nullable*/, int n_masks, const double* ps,
                         int n_p, double* means, long long* counts, long long* status, long long* scratch, void* stream);

/* ---- POT threshold of eval_methods.py pot_eval (spot.py SPOT: initialize, _grimshaw, _quantile, run(with_alarm=False))
 *      on device floats init (n_init training scores) and data (n test scores).  t = the k-th smallest of init (exact;
 *      k = int(level * n_init) after level -= floor(level), computed by the caller; -0.0 orders before +0.0); the peaks
 *      are init[init > t] - t; the Grimshaw fit returns the maximum-likelihood candidate among the outermost nodes
 *      with a finite w of spot.py's two search intervals and the roots of w found by bisecting the sign changes of w over 353 nodes per interval
 *      (DESIGN §1).  dynamic = 1: SPOT.run's refits, one per test point x > t, all in parallel; valid while no point
 *      x <= t lies above the previous extreme quantile (checked: status[2]).
 *      out: 10 device words, doubles out[0..5] = {t, pot_th, gamma, sigma, ll, z} (gamma .. z of the initial fit, z = 0
 *      for the gamma = 0 baseline; pot_th = the static quantile, or the mean of the per-point thresholds), then int64
 *      status[0..3] = {initial peaks, refits, first index where the dynamic premise fails or -1, MTADGAT_POT_* flags}.
 *      thresholds (nullable): n device doubles, the extreme quantile recorded for each test point.
 *      scratch: mtadgat_pot_scratch_bytes(n_init, n) bytes, 8-byte aligned.  n_init + n < 2^31.  No allocation, no
 *      synchronisation, no floating-point atomics (CUDA-graph capturable, run-to-run identical). ---- */
#define MTADGAT_POT_NAN 1          /* a score is NaN */
#define MTADGAT_POT_NO_PEAKS 2     /* no training score above t (spot.py: peaks.min() of an empty array) */
#define MTADGAT_POT_EQUAL_PEAKS 4  /* all initial peaks equal (spot.py: np.arange with a zero step) */
#define MTADGAT_POT_BASELINE 8     /* every fit chose gamma = 0: every recorded threshold is a float32 */
long long mtadgat_pot_scratch_bytes(long long n_init, long long n);
int mtadgat_pot(const float* init, long long n_init, const float* data, long long n, long long k, double q, int dynamic,
                double* out, double* thresholds /*nullable*/, void* scratch, void* stream);

/* ---- streaming SPOT (spot.py SPOT.initialize + SPOT.run(dynamic=True) point by point, either with_alarm) on a
 *      caller-allocated device state of MTADGAT_SPOT_STATE_WORDS int64 words and a device float peak array it points to.
 *      mtadgat_spot_stream_init (spot.py SPOT.initialize): t = the k-th smallest of init as in
 *      mtadgat_pot, the peaks init[init > t] - t in float32, in index order, into `peaks` (capacity >= n_init - k floats),
 *      the initial Grimshaw fit with n = n_init and its extreme quantile.  scratch:
 *      mtadgat_spot_stream_init_scratch_bytes(n_init) bytes, 8-byte aligned; only the init launches use it.
 *      mtadgat_spot_stream_push (the dynamic branch of spot.py SPOT.run's loop): for each of the m scores in order,
 *      x > quantile: an alarm with with_alarm (nothing else changes), else a new peak; t < x <= quantile: a new peak;
 *      otherwise n += 1.  A new peak appends x - t (float32; <= 0 is possible when the quantile is below t), increments
 *      Nt and n, and refits over all Nt peaks.  thresholds[i] = the quantile after point i (double), alarms[i] = 0 / 1.
 *      Scores are compared as numpy compares them: x > t in float32, x > quantile in double.
 *      mtadgat_spot_stream_grow moves the peaks to a new array of `capacity` floats (the caller keeps the capacity at
 *      least Nt + m before each push; the push stops with MTADGAT_POT_CAPACITY instead of writing past it).
 *      Errors are sticky: once a flag is set (NaN score, no initial peaks, all peaks equal, a mean peak <= 0, capacity), a
 *      push processes nothing; the points a push did not process get a NaN threshold and no alarm.
 *      No allocation, no synchronisation, no floating-point atomics (CUDA-graph capturable, run-to-run identical). ---- */
#define MTADGAT_POT_CAPACITY 16    /* streaming SPOT: a new peak did not fit in the peak array */
#define MTADGAT_POT_NONPOSITIVE_MEAN 32  /* streaming SPOT: the mean peak is <= 0 (spot.py: math.log of it raises) */
#define MTADGAT_SPOT_STATE_WORDS 24
#define MTADGAT_SPOT_T 0           /* double: t (a float32 value) */
#define MTADGAT_SPOT_N 1           /* int64: n, points observed (training scores included) */
#define MTADGAT_SPOT_NT 2          /* int64: Nt, peaks */
#define MTADGAT_SPOT_QUANTILE 3    /* double: the current extreme quantile */
#define MTADGAT_SPOT_FLAGS 4       /* int64: MTADGAT_POT_* flags */
#define MTADGAT_SPOT_PEAKS 5       /* int64: device address of the peak array */
#define MTADGAT_SPOT_CAPACITY 6    /* int64: its capacity in floats */
#define MTADGAT_SPOT_Q 7           /* double: q (spot.py's proba) */
#define MTADGAT_SPOT_ALARMS 8      /* int64: alarms of the last push */
#define MTADGAT_SPOT_JOINED 9      /* int64: peaks added by the last push */
#define MTADGAT_SPOT_DONE 10       /* int64: points the last push processed (m unless it stopped on an error) */
#define MTADGAT_SPOT_FIT 11        /* doubles [11, 17): the last fit {quantile, gamma, sigma, ll, z, all-equal flag} */
long long mtadgat_spot_stream_init_scratch_bytes(long long n_init);
int mtadgat_spot_stream_init(const float* init, long long n_init, long long k, double q, long long* state, float* peaks,
                             long long capacity, void* scratch, void* stream);
/* SPOT.initialize of n_streams independent streams in one launch sequence whose length does not depend on n_streams
 * (thresholding.SpotStreams, when a fleet is built and when streams are added to it).  init: the streams' training
 * scores concatenated, n_total floats; offsets: n_streams + 1 device int64, rising from 0 to n_total, every stream with
 * at least one score (stream s owns init[offsets[s] : offsets[s+1]]); ks: n_streams device int64, stream s's rank
 * (0 <= ks[s] < its length); states: n_streams consecutive MTADGAT_SPOT_STATE_WORDS blocks; peaks: 2 * n_streams device
 * int64, stream s's peak array {device address, capacity in floats}.  The tables are trusted.  Every stream's state
 * block and peaks are bitwise what mtadgat_spot_stream_init writes for it alone (that entry point is the one-stream case
 * of this one), apart from the peak address and capacity words; a stream whose peaks would exceed its capacity gets
 * MTADGAT_POT_CAPACITY and no peaks.  scratch: mtadgat_spot_stream_init_batched_scratch_bytes(n_total, n_streams)
 * bytes, 8-byte aligned.  n_total < 2^31.  No allocation, no synchronisation, no floating-point atomics. */
long long mtadgat_spot_stream_init_batched_scratch_bytes(long long n_total, int n_streams);
int mtadgat_spot_stream_init_batched(const float* init, long long n_total, const long long* offsets, const long long* ks,
                                     int n_streams, double q, long long* states, const long long* peaks, void* scratch,
                                     void* stream);
int mtadgat_spot_stream_grow(long long* state, float* peaks, long long capacity, void* stream);
int mtadgat_spot_stream_push(long long* state, const float* scores, long long m, int with_alarm, double* thresholds,
                             unsigned char* alarms, void* stream);
/* the same push for n_streams independent streams in one launch (thresholding.SpotStreams): `states` is n_streams
 * consecutive MTADGAT_SPOT_STATE_WORDS blocks, each filled by mtadgat_spot_stream_init or _init_batched (its own peak
 * array) and grown by mtadgat_spot_stream_grow on that block; offsets: n_streams + 1 device int64, non-decreasing from 0; stream s
 * walks scores[offsets[s] : offsets[s+1]] and writes the same slice of thresholds / alarms and its own block, one CTA
 * per stream.  A stream with no scores, or with an error flag already set, processes nothing (DONE = 0; its slice gets
 * NaN thresholds and no alarms); a stream's error stops that stream only.  Every stream's results are bitwise those of
 * mtadgat_spot_stream_push on its block and slice alone. */
int mtadgat_spot_stream_push_batched(long long* states, int n_streams, const float* scores, const long long* offsets,
                                     int with_alarm, double* thresholds, unsigned char* alarms, void* stream);

/* ---- streaming dSPOT (spot.py backMean + dSPOT.initialize + dSPOT.run, SPOT with drift) on the state blocks of the
 *      streaming SPOT above plus one window of the last `depth` normal scores per stream, (n_streams, depth) float32,
 *      oldest first.  1 <= depth <= MTADGAT_DSPOT_MAX_DEPTH.
 *      mtadgat_dspot_residuals_batched (spot.py backMean(init, d) and dSPOT.initialize's T = init[d:] - M[:-1]):
 *      init and offsets as mtadgat_spot_stream_init_batched takes them, every stream with more than depth scores;
 *      stream s's n_s - depth residuals go to resid[offsets[s] - s * depth ...] (n_total - n_streams * depth floats)
 *      and its last depth scores to windows[s].  The moving sum starts as numpy's pairwise sum of the first depth
 *      scores and moves one float32 subtraction and addition at a time, as backMean's loop does.  The caller then runs
 *      mtadgat_spot_stream_init_batched on the residuals (offsets minus s * depth, ks = int(level * (n_s - depth))):
 *      dSPOT.initialize's t, peaks and first fit, with n = n_s - depth.
 *      mtadgat_dspot_push_batched (dSPOT.run's loop): as mtadgat_spot_stream_push_batched, with Mi = W.mean() (numpy's
 *      pairwise float32 sum of the window, divided by depth) and r = x - Mi in place of x: r > quantile is an alarm
 *      (with_alarm: W and n unchanged) or else a peak r - t; t < r <= quantile a peak; a point that is not an alarm
 *      replaces the oldest score of W.  thresholds[i] = quantile + Mi after point i, in double, or in float32 while the
 *      quantile is the gamma = 0 baseline (fit word gamma = 0).  offsets null: one stream of m scores.  Each CTA
 *      stages its window in shared memory and writes it back oldest first.  Stop flags, capacity (grow with
 *      mtadgat_spot_stream_grow) and status words are those of mtadgat_spot_stream_push_batched.
 *      No allocation, no synchronisation, no floating-point atomics. ---- */
#define MTADGAT_DSPOT_MAX_DEPTH 4096
int mtadgat_dspot_residuals_batched(const float* init, long long n_total, const long long* offsets, int n_streams,
                                    int depth, float* resid, float* windows, void* stream);
int mtadgat_dspot_push_batched(long long* states, int n_streams, float* windows, int depth, const float* scores,
                               const long long* offsets, long long m, int with_alarm, double* thresholds,
                               unsigned char* alarms, void* stream);

/* ---- streaming biSPOT / bidSPOT (spot.py's two-sided SPOT, and two-sided SPOT with drift) on two state blocks per
 *      stream: `upper` and `lower`, each n_streams consecutive MTADGAT_SPOT_STATE_WORDS blocks with their own peak
 *      arrays.  The lower side is SPOT on the negated scores: its block holds -t_down, -Q_down and the peaks
 *      t_down - x, so the caller initialises it with mtadgat_spot_stream_init_batched on -x (bidSPOT: on the negated
 *      residuals of mtadgat_dspot_residuals_batched) at rank n - 1 - int((1 - level) n).  Both blocks start with the
 *      same N, which stays shared.
 *      mtadgat_bispot_push_batched (biSPOT.run / bidSPOT.run's loop): for each score, r = x (depth 0) or x - W.mean()
 *      (1 <= depth <= MTADGAT_DSPOT_MAX_DEPTH, windows as mtadgat_dspot_push_batched takes them), the first of:
 *      r > Q_up an alarm (with_alarm) or else an upper peak; r > t_up an upper peak; r < Q_down an alarm or else a
 *      lower peak; r < t_down a lower peak; otherwise n += 1.  A peak refits its own side only, with the shared n.
 *      Every point but an alarm enters W.  upper_thresholds[i] / lower_thresholds[i] = Q_up / Q_down after point i
 *      (with a depth: plus Mi, as mtadgat_dspot_push_batched records it, per side); alarms[i] = 0 none, 1 above,
 *      2 below.  offsets null: one stream of m scores.  A stop flag on either side stops the stream and the same
 *      FLAGS word is written to both blocks, as is DONE; ALARMS, JOINED and FIT are per side.  Capacity (grow each
 *      block with mtadgat_spot_stream_grow), NaN scores and the unprocessed tail are mtadgat_spot_stream_push_batched's.
 *      mtadgat_spot_state_export / _import: the state blocks and peaks of B streams, mtadgat_stream_state_export /
 *      _import's SPOT part alone (the lower half of a two-sided record).  tab (device int64, trusted): slot[B],
 *      poff[B + 1] as there; for an import, then {address, capacity} of each stream's new peak array.  Export zeroes
 *      PEAKS and CAPACITY; import sets them from the table.  One launch each, bit copies only.
 *      No allocation, no synchronisation, no floating-point atomics. ---- */
int mtadgat_bispot_push_batched(long long* upper, long long* lower, int n_streams, float* windows, int depth,
                                const float* scores, const long long* offsets, long long m, int with_alarm,
                                double* upper_thresholds, double* lower_thresholds, unsigned char* alarms,
                                void* stream);

/* ---- one push for n_streams streams that each run their own rule (thresholding.SpotStreams with configs): SPOT,
 *      dSPOT, biSPOT or bidSPOT per stream, with its own depth and with_alarm, one CTA per stream in one launch.
 *      states: 2 * n_streams MTADGAT_SPOT_STATE_WORDS blocks, the (2, S, 24) layout mtadgat_bispot_push_batched takes
 *      as upper = states, lower = states + S blocks: stream s's block is s and, two-sided, its lower block S + s (a
 *      one-sided stream's lower block is never read or written).  Each block is initialised and grown as for its
 *      rule's own push.  tab: MTADGAT_MIXED_WORDS device int64 per stream (trusted) = {rule (MTADGAT_RULE_*), depth
 *      (0 for SPOT / biSPOT, 1 .. MTADGAT_DSPOT_MAX_DEPTH otherwise), the offset in floats of its window in `windows`
 *      (depth floats, oldest first; unused without a depth), with_alarm}.  windows: the streams' windows in one ragged
 *      float32 buffer (nullable when no stream has a depth).  offsets: n_streams + 1 device int64, non-decreasing from
 *      0; stream s walks scores[offsets[s] : offsets[s+1]] with the push body of its rule (mtadgat_spot_stream_push,
 *      mtadgat_dspot_push_batched, mtadgat_bispot_push_batched without / with a depth) and writes the same slice of
 *      upper_thresholds, lower_thresholds (NaN for a one-sided stream) and alarms (uint8: 0 none, 1 above, 2 below).
 *      Every stream's results, state words and window are bitwise those of its rule's push on it alone.
 *      No allocation, no synchronisation, no floating-point atomics. ---- */
#define MTADGAT_RULE_SPOT 0
#define MTADGAT_RULE_DSPOT 1
#define MTADGAT_RULE_BISPOT 2
#define MTADGAT_RULE_BIDSPOT 3
#define MTADGAT_MIXED_RULE 0
#define MTADGAT_MIXED_DEPTH 1
#define MTADGAT_MIXED_WINDOW 2
#define MTADGAT_MIXED_ALARM 3
#define MTADGAT_MIXED_WORDS 4
int mtadgat_spot_mixed_push_batched(long long* states, int n_streams, const long long* tab, float* windows,
                                    const float* scores, const long long* offsets, double* upper_thresholds,
                                    double* lower_thresholds, unsigned char* alarms, void* stream);
/* ---- a replay over many labelled streams (thresholding.replay_streams, and thresholding.replay with one stream):
 *      n_walks walks of mixed rules, each over its own slice of one concatenated score array, one CTA per walk, one
 *      launch per chunk [lo, lo + chunk).  tab: MTADGAT_FLEET_REPLAY_WORDS device int64 per walk (trusted); its first
 *      four words are a MTADGAT_MIXED_* row (rule, depth, window offset in `windows`, with_alarm), then the walk's
 *      upper and lower state blocks (indices of MTADGAT_SPOT_STATE_WORDS blocks in `states`; the lower one is read and
 *      written by two-sided rules only), the offset and length m_j of its score slice, and the offsets of its alarm row
 *      and of its upper and lower threshold rows.  Walk j covers points [lo, min(lo + chunk, m_j)) of its slice, point
 *      lo + k at index k of every pointer argument plus the table's offset: the caller passes scores, alarms and
 *      full-length threshold buffers advanced by lo (elements), or a threshold buffer of chunk-sized scratch rows that
 *      every chunk reuses as it is.  A walk whose slice ended at or before lo returns and writes nothing.  Each walk
 *      runs its rule's push body, as mtadgat_spot_mixed_push_batched does (one-sided walks write NaN lower thresholds),
 *      so its thresholds, alarms, window and block words are bitwise those of its rule's push on that block alone,
 *      except ALARMS, JOINED and DONE: the walk adds the values the block held before, so after the last chunk every
 *      block holds the words of one push of the whole slice.  Stop flags, NaN scores and the capacity check are the
 *      push's; a walk's error stops that walk only.  The caller keeps each peak array's capacity at least Nt + m_j (no
 *      grow here).  No allocation, no synchronisation, no floating-point atomics. ---- */
#define MTADGAT_FLEET_REPLAY_UPPER 4
#define MTADGAT_FLEET_REPLAY_LOWER 5
#define MTADGAT_FLEET_REPLAY_SCORES 6
#define MTADGAT_FLEET_REPLAY_LENGTH 7
#define MTADGAT_FLEET_REPLAY_ALARMS 8
#define MTADGAT_FLEET_REPLAY_THR_UP 9
#define MTADGAT_FLEET_REPLAY_THR_LO 10
#define MTADGAT_FLEET_REPLAY_WORDS 11
int mtadgat_spot_fleet_replay(long long* states, int n_walks, const long long* tab, float* windows,
                              const float* scores, long long lo, long long chunk, double* upper_thresholds,
                              double* lower_thresholds, unsigned char* alarms, void* stream);
int mtadgat_spot_state_export(const long long* states, const long long* tab, int n_streams, long long max_peaks,
                              long long* words, float* peaks_out, void* stream);
int mtadgat_spot_state_import(const long long* words, const float* peaks_in, const long long* tab, int n_streams,
                              long long max_peaks, long long* states, void* stream);

/* ---- scoring many live streams with one model (scoring.MultiStreamScorer): S streams, each with a ring of its last n
 *      rows, hist (S, n, k) with hist[s][g % n] = row g of stream s, and the forecast of its last window, last_preds
 *      (S, out).  A push brings R new rows of any mix of streams as one (R, k) array `rows`; the index tables are device
 *      int64, built on the host (scoring.fleet_tables) and trusted.  `perm` (R): the rows' positions grouped by stream in
 *      arrival order (sorted position -> row of `rows`).
 *      mtadgat_gather_stream_windows: x[b] (n*k floats), b < count, = rows first .. first + n - 1 of stream s, with
 *      tab (4, ld) = {s, first, n_old, xpos} per window: the first n_old rows come from the ring, the others are
 *      rows[perm[xpos ..]].  A window never reads another stream's rows.
 *      mtadgat_score_epilogue_indexed: mtadgat_score_epilogue's per-feature arithmetic for m completed timestamps with
 *      tab (3, ld) = {f, r, a}: forecast[i] = preds[f] (f >= 0) or last_preds[-1 - f], recon[i] = recons_last[r], actual
 *      = rows[a][target_dims ? target_dims[c] : c]; forecast, recon, actual, a_score are (m, out) outputs.  The global
 *      score is mtadgat_row_mean of a_score.
 *      mtadgat_stream_history_update, after the two above: hist row row_tab[n_rows + p] (skipped when < 0) =
 *      rows[row_tab[p]], p < n_rows, and last_preds[pred_tab[n_preds + j]] = preds[pred_tab[j]], j < n_preds; destinations
 *      are distinct.  No allocation, no synchronisation, no atomics (CUDA-graph capturable). ---- */
int mtadgat_gather_stream_windows(const float* rows, const float* hist, const long long* perm, const long long* tab,
                                  long long ld, int count, int n, int k, float* x, void* stream);
int mtadgat_score_epilogue_indexed(const float* preds, const float* last_preds, const float* recons_last,
                                   const float* rows, const long long* tab, long long ld, const int* target_dims, int k,
                                   int out, long long m, float gamma, float* forecast, float* recon, float* actual,
                                   float* a_score, void* stream);
int mtadgat_stream_history_update(const float* rows, const long long* row_tab, long long n_rows, const float* preds,
                                  const long long* pred_tab, long long n_preds, int k, int out, float* hist,
                                  float* last_preds, void* stream);

/* ---- the live state of B streams as one portable record (prediction.FleetDetector / StreamDetector.state_dict and
 *      from_state_dict).  Per record stream b: words (B, MTADGAT_SPOT_STATE_WORDS) int64, hist_rec (B, n, k) with row
 *      j < h = min(rows[b], n) = the stream's row rows[b] - h + j (chronological) and the rows after h zero, pred_rec
 *      (B, out) = its last window's forecast (zero while rows[b] < n), and peaks_rec[poff[b] : poff[b+1]] = its first Nt
 *      peaks.  A detector's history is a ring (layout MTADGAT_STREAM_RING: row g of stream s at hist[s][g % n], hist
 *      (S, n, k)) or linear (MTADGAT_STREAM_LINEAR: chronological row j at hist[s][j], as StreamDetector keeps it).
 *      tab (device int64, trusted): slot[B] (the detector's stream of record stream b), rows[B], poff[B + 1]
 *      non-decreasing from 0 with poff[b+1] - poff[b] = that stream's Nt; for an import, then {address, capacity} of
 *      each stream's new peak array (capacity >= Nt), as mtadgat_spot_stream_init_batched takes them.  max_peaks >= the
 *      largest Nt (it sizes the grid).
 *      mtadgat_stream_state_export: writes the record of the B streams; the state words' PEAKS and CAPACITY are zeroed,
 *      every other word is copied, and the peaks are read through each block's PEAKS address.  hist may be null when
 *      every rows[b] is 0, last_preds when none reaches n.
 *      mtadgat_stream_state_import: writes the B streams' histories (a ring gets all n rows, a linear history its h),
 *      last forecasts (skipped when last_preds is null), state blocks (PEAKS and CAPACITY from the table) and peaks.
 *      One launch each; both only copy bits (no floating-point arithmetic), allocate nothing and do not synchronise. */
#define MTADGAT_STREAM_RING 0
#define MTADGAT_STREAM_LINEAR 1
int mtadgat_stream_state_export(const float* hist, const float* last_preds, const long long* states,
                                const long long* tab, int n_streams, int n, int k, int out, int layout,
                                long long max_peaks, long long* words, float* hist_rec, float* pred_rec,
                                float* peaks_rec, void* stream);
int mtadgat_stream_state_import(const long long* words, const float* hist_rec, const float* pred_rec,
                                const float* peaks_rec, const long long* tab, int n_streams, int n, int k, int out,
                                int layout, long long max_peaks, float* hist, float* last_preds, long long* states,
                                void* stream);

/* ---- per-feature streaming SPOT (prediction's detectors with per_feature=True): feature i of stream s is SPOT stream
 *      s*out + i of the streaming SPOT / dSPOT / biSPOT kernels above, whose pushes take each stream's scores as one
 *      contiguous run.  A push's m scores (m, out) row-major are grouped by stream: streams (m, device int64) names the
 *      stream of each row and offsets (n_streams + 1, device int64, non-decreasing from 0 to m) delimits each stream's
 *      rows, as MultiStreamScorer's push returns them (trusted); both null: the m rows are one stream (n_streams 1).
 *      mtadgat_feature_gather: scores[out*off[s] + i*m_s + (r - off[s])] = a_score[r*out + i] for row r of stream s
 *      (m_s = off[s+1] - off[s]), and feature_offsets (n_streams*out + 1 int64) = the start of each feature stream's
 *      run, out*off[s] + i*m_s, then m*out.
 *      mtadgat_feature_scatter: the inverse map for a push's results: thresholds_out / lower_out (m, out) doubles and
 *      alarms_out (m, out) bytes (bool, or biSPOT's codes) from the feature-major thresholds / lower_thresholds (both
 *      null, or neither) / alarms.
 *      One launch each; both move raw bits only, allocate nothing and do not synchronise. ---- */
int mtadgat_feature_gather(const float* a_score, long long m, int out, const long long* streams,
                           const long long* offsets, int n_streams, float* scores, long long* feature_offsets,
                           void* stream);
int mtadgat_feature_scatter(const double* thresholds, const double* lower_thresholds, const unsigned char* alarms,
                            long long m, int out, const long long* streams, const long long* offsets,
                            double* thresholds_out, double* lower_out, unsigned char* alarms_out, void* stream);

/* ---- per-feature robust scaling of the anomaly scores, Predictor.get_score's scale_scores=True (prediction.py:82-86):
 *      for each column sc of the row-strided (n, C) device float32 matrix a (column c is a[i*ld + c], ld >= C),
 *      stats[3c ..] = {m = np.median(sc) (a float32 value), q25, q75 = np.percentile(sc, [25, 75])} (doubles), from
 *      exact order statistics (-0.0 orders before +0.0); scaled (n, C) doubles = (sc - m) / (1 + (q75 - q25)) with the
 *      difference in float32 and the quotient in double; global[i] (n floats) = np.mean of row i of scaled rounded to
 *      float32, in numpy's pairwise summation order.  A NaN in a column makes its statistics (and so its scaled values)
 *      NaN.  All bitwise equal to numpy.  scratch: mtadgat_robust_scale_scratch_bytes(n, C) bytes, 8-byte aligned.
 *      C <= 65535.  No allocation, no synchronisation, no floating-point atomics (CUDA-graph capturable). ---- */
long long mtadgat_robust_scale_scratch_bytes(long long n, int C);
int mtadgat_robust_scale(const float* a, long long n, int C, long long ld, double* stats, double* scaled, float* global,
                         void* scratch, void* stream);
/* out[i] (n floats) = np.mean(a, 1)[i] of the row-strided (n, C) device float32 matrix a, bitwise: numpy's pairwise
 * summation order from +0.0, then / C in float32 (get_score's unscaled A_Score_Global). */
int mtadgat_row_mean(const float* a, long long n, int C, long long ld, float* out, void* stream);

/* ---- SMAP / MSL channel adjustment of a global anomaly score (utils.py adjust_anomaly_scores, the part after the channel
 *      metadata is read).  out = scores with out[zero_idx[t]] = +0.0 (n_zero device int64 indices; those outside
 *      [0, n) are skipped); then for j = 0 .. n_bounds-2 in order, the slice out[bounds[j] : bounds[j+1] + 1] (clipped
 *      to n) becomes (e - min(e)) / (max(e) - min(e)) in float32.  Consecutive slices share bounds[j+1]: it is
 *      normalised by segment j, then again by segment j+1, whose min / max include its normalised value.  bounds:
 *      n_bounds device int64, strictly increasing, bounds[j] < n for j < n_bounds - 1 (every slice non-empty; the
 *      caller checks).  min / max propagate NaN (a NaN makes its segment NaN); max == min gives NaN (0 / 0).  Bitwise
 *      numpy's results, except that a zero result may carry either sign.  out may alias scores.  scratch:
 *      mtadgat_channel_adjust_scratch_bytes(n, n_bounds) bytes, 4-byte aligned.  n_bounds - 1 <= 65535.  No
 *      allocation, no synchronisation, no floating-point atomics (CUDA-graph capturable). ---- */
long long mtadgat_channel_adjust_scratch_bytes(long long n, int n_bounds);
int mtadgat_channel_adjust(const float* scores, long long n, const long long* zero_idx, long long n_zero,
                           const long long* bounds, int n_bounds, float* out, void* scratch, void* stream);

/* ---- recurrence implementation: 1 (default) = persistent warpgroup-MMA kernel, fp16 operands with fp32
 *      accumulation and fp32 hidden state (hidden sizes 8..256); 0 = fp32 SIMT kernel.  mtadgat_tc_probe runs one
 *      mma_m x N x K product (mma_m = 64 or 128, D row-major) through the same shared-memory operand layout
 *      (diagnostic / unit test). ---- */
int mtadgat_set_gru_impl(int impl);
int mtadgat_get_gru_impl(void);
/* cluster recurrence: clusters per 16-window tile, 0 = auto (default; small batches split a tile over 2 or 4
 * clusters so that more SMs work on the serial chain), or 1 / 2 / 4.  Results do not depend on it. */
int mtadgat_set_gru_split(int split);
/* cluster BPTT variant: 0 (default) = unit split (every CTA multiplies the whole dgh vector for its units: 30 MMAs per
 * step), 1 = K split over the cluster (each CTA multiplies its own gate slice for all units, fp32 partial sums exchanged
 * over DSMEM: a shorter MMA chain, but two hand-offs per step).  Same results. */
int mtadgat_set_gru_bptt(int ksplit);
/* The recurrence alone (torch.nn.GRU's per-step part, modules.py:235-238) on WINDOW-TILED internals
 * T[b/16][t][channel][b%16] (B rounded up to 16): gi_t = x W_ih^T + b_ih (channels 3H), gates_t (4H: r,z,n,h_n),
 * dgi_t (3H), dghn_t (H).  mtadgat_gru_fwd / _bwd = projection GEMMs + these.  wt_scratch: 3H*H floats;
 * gmax_word: one device word.  bench.py times these entry points for the per-kernel roofline. */
int mtadgat_gru_recurrence_fwd(const float* gi_t, const float* w_hh, const float* b_hh, float* wt_scratch, float* out,
                               float* h_last /*nullable*/, float* gates_t /*nullable*/, int B, int n, int H, void* stream);
int mtadgat_gru_recurrence_bwd(const float* gates_t, const float* out, const float* w_hh, const float* dout /*nullable*/,
                               const float* dh_last /*nullable*/, float* dgi_t, float* dghn_t, unsigned int* gmax_word,
                               int B, int n, int H, void* stream);
/* GEMM-shaped stages (conv, projections, heads, weight gradients): 1 (default) = warpgroup MMAs on bf16 hi/lo splits
 * (bf16x3, ~1e-5 relative) from operands packed into a per-stream workspace, 0 = SIMT fp32. */
int mtadgat_set_gemm_impl(int impl);
int mtadgat_get_gemm_impl(void);
/* The packed-operand GEMM keeps ONE grow-only device buffer per stream it is called on (the only memory the library
 * owns; the fixed-order reductions use it as scratch too).  It grows on demand, except while the stream is being captured into a CUDA graph: run the same call eagerly
 * once on that stream first, or reserve it here.  A buffer that a capture has used is never freed when the workspace
 * later grows (replays of that graph stay valid).  _release frees every buffer (synchronises the device; graphs
 * captured before it must not be replayed afterwards). */
int mtadgat_workspace_reserve(void* stream, long long bytes);
void mtadgat_workspace_release(void);
int mtadgat_tc_probe(const float* A, const float* Bm, float* D, int Mtot, int row0, int K, int N, int b_mn_major,
                     int mma_m, void* stream);
/* optional: per-phase cycle counters of the cluster GRU (forward and unit-split BPTT).  dev_ptr holds `slots` slots of
 * 16 int64; each launch fills the next slot, round robin from slot 0 (layout in csrc/gru_cl.cu).  While set, the
 * launches run the instrumented kernel variants.  slots = 0 turns it off. */
void mtadgat_gru_debug_buffer(long long* dev_ptr, int slots);

/* ---- CPU backend (host pointers, synchronous, fp32, OpenMP over windows): the same stages for tensors that live on the
 *      host -- the reference's callers pick the device from the tensors (training.py:60, prediction.py:45).  Selected by the tensors' device; CUDA tensors never come
 *      here.  att (B,K,K): softmax output, written when non-null and required by the backward; gates (B,n,4H) likewise.
 *      Dropout uses the same Philox streams as the CUDA kernels, seeded by value. ---- */
int mtadgat_cpu_conv_relu_fwd(const float* x, const float* w, const float* bias, float* y, int B, int n, int k, int ks);
int mtadgat_cpu_conv_relu_bwd(const float* x, const float* w, const float* y, const float* dy, float* dx /*nullable*/,
                              float* dw, float* db, int B, int n, int k, int ks);
int mtadgat_cpu_gat_fwd(const float* x, const float* lin_w, const float* lin_b, const float* a, const float* bias,
                        float* out, float* att /*nullable*/, int B, int n, int k, int E, int feature, int use_gatv2,
                        float alpha, float p_drop, unsigned long long seed);
int mtadgat_cpu_gat_bwd(const float* x, const float* lin_w, const float* lin_b, const float* a, const float* att,
                        const float* out, const float* gout, float* dx, float* dlin_w, float* dlin_b, float* da,
                        float* dbias /*nullable*/, int B, int n, int k, int E, int feature, int use_gatv2, float alpha,
                        float p_drop, unsigned long long seed);
int mtadgat_cpu_gru_fwd(const float* x, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                        float* out, float* gates /*nullable*/, int B, int n, int I, int H);
int mtadgat_cpu_gru_bwd(const float* x, const float* w_ih, const float* w_hh, const float* out, const float* gates,
                        const float* dout, float* dx /*nullable*/, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh,
                        int B, int n, int I, int H);
int mtadgat_cpu_linear_fwd(const float* x, const float* w, const float* b, float* y, int M, int I, int O, int act,
                           float p_drop, unsigned long long seed, unsigned int rng_stream);
int mtadgat_cpu_linear_bwd(const float* x, const float* w, const float* y, const float* dy, float* dx /*nullable*/,
                           float* dw, float* db, int M, int I, int O, int act, float p_drop, unsigned long long seed,
                           unsigned int rng_stream);

/* ---- RNG plumbing ---- */
int mtadgat_dropout_mask(float* out, long long numel, float p, const unsigned long long* seed,
                         unsigned int rng_stream, void* stream);   /* multipliers 0 or 1/(1-p), for tests */
int mtadgat_seed_advance(unsigned long long* seed, void* stream);  /* new seed per step, on device */

#ifdef __cplusplus
}
#endif
#endif /* MTADGAT_H_ */
