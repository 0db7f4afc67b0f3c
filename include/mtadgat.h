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

#define MTADGAT_ABI_VERSION 1

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
/* GAT forward structure for layers whose window fits one CTA (K <= 128 nodes): 0 (default) = projection GEMM to HBM +
 * score kernel; 1 = ONE fused kernel per layer (in-kernel tensor-core projection of the window from packed weights, P/Q
 * kept in shared memory, score, softmax, dropout, aggregation, sigmoid).  Results are identical. */
int mtadgat_set_gat_impl(int impl);
int mtadgat_get_gat_impl(void);
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
 * (bf16x3, ~1e-5 relative) from operands packed into a per-stream workspace, 2 = same arithmetic with the operand
 * gather inside the GEMM kernel (no workspace), 0 = SIMT fp32. */
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
void mtadgat_gru_debug_buffer(long long* dev_ptr);   /* optional: 16 int64 per-phase cycle counters of the cluster GRU */

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
