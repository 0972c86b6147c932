/*
 * kge_b200.h — C-ABI of the H100-native (sm_90a) KGE scoring engine (libkge_b200.so).
 *
 * The reference (Sujit-O/pykg2vec) has NO native interface: its hot path is the
 * duck-typed Python surface `model.forward(h, r, t)` / `model.loss(...)` /
 * `Evaluator.test_*_rank` executed as chains of ATen ops.  Each entry point
 * below replaces one such chain; the comment above it cites the reference
 * lines (relative to /root/reference/) whose behaviour it reproduces.
 *
 * Conventions
 *   - plain `extern "C"`, POD arguments, raw DEVICE pointers unless the name
 *     says `host`; no torch / C++ types cross this boundary.
 *   - every function returns 0 on success, a negative KGE_E* code otherwise and
 *     never throws; `kge_last_error()` returns a thread-local message.
 *   - nothing is allocated or retained: all buffers are borrowed for the call,
 *     outputs and workspaces are pre-allocated by the caller.
 *   - `stream` is a `cudaStream_t` passed as `void*` (0 = legacy default
 *     stream).  All work is enqueued asynchronously on it.
 *   - no CUDA state is touched at load time (fork-safe: pykg2vec forks sampler
 *     processes after CUDA init, pykg2vec/data/generator.py:292-312).
 *   - ids are int64 (torch.LongTensor, pykg2vec/utils/trainer.py:275-293),
 *     tables are fp32 row-major [rows, dim] (nn.Embedding weights,
 *     pykg2vec/models/Domain.py:8-17), scores are fp32.
 *
 * Canonical arithmetic ("RSUM order") is specified in DESIGN.md §3; the CPU
 * oracle (oracle/kge_oracle.c) restates it independently and the two agree
 * bit-for-bit on scores and therefore exactly on ranks.
 */
#ifndef KGE_B200_H
#define KGE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KGE_ABI_VERSION 10
#define KGE_MAX_TABLES 16

/* status codes */
#define KGE_OK 0
#define KGE_EINVAL -1   /* bad argument (null pointer, unsupported dim, ...) */
#define KGE_ENOTSUP -2  /* model / mode not implemented by this entry point */
#define KGE_ECUDA -3    /* CUDA runtime error, see kge_last_error() */
#define KGE_EWORKSPACE -4 /* workspace too small */

/* model ids.  Table order in kge_model_t.tables[] is given per model.
 * (file:line = the reference forward()/embed() being replaced) */
enum kge_model_id {
  KGE_TRANSE = 0,   /* [ent, rel]                       pairwise.py:56-93   */
  KGE_TRANSH = 1,   /* [ent, rel, w]                    pairwise.py:143-182 */
  KGE_TRANSD = 2,   /* [ent, rel, ent_map, rel_map]     pairwise.py:229-278 */
  KGE_TRANSR = 3,   /* [ent, rel, rel_matrix]           pairwise.py:405-470 */
  KGE_ROTATE = 4,   /* [ent_re, ent_im, rel]            pairwise.py:765-791 */
  KGE_HOLE = 5,     /* [ent, rel]  (as evaluated by torch<1.7) pairwise.py:1119-1125 */
  KGE_DISTMULT = 6, /* [ent, rel]                       pointwise.py:444-446 */
  KGE_COMPLEX = 7,  /* [ent_re, ent_im, rel_re, rel_im] pointwise.py:163-188 */
  KGE_CP = 8,       /* [sub, rel, obj]                  pointwise.py:374-376 */
  KGE_SIMPLE = 9,   /* [ent_h, ent_t, rel, rel_inv]     pointwise.py:522-526 */
  KGE_TRANSM = 10,  /* [ent, rel, theta(R x 1)]         pairwise.py:325-347 */
  KGE_RESCAL = 11,  /* [ent, rel_matrices(R x d*d)]     pairwise.py:829-865 */
  KGE_ANALOGY = 12, /* [ent, rel, ent_re, ent_im, rel_re, rel_im] (re/im half width) pointwise.py:97-104 */
  KGE_SIMPLE_IGNR = 13, /* [ent_h, ent_t, rel, rel_inv]  pointwise.py:573-581 */
  KGE_QUATE = 14,   /* [ent_s, ent_x, ent_y, ent_z, rel_s, rel_x, rel_y, rel_z]  pointwise.py:678-694 */
  KGE_OCTONIONE = 15, /* [ent_1..ent_8, rel_1..rel_8]   pointwise.py:886-899 */
  KGE_KG2E = 16,    /* [ent_mu, ent_sigma, rel_mu, rel_sigma] pairwise.py:1021-1084 */
  /* dense-layer models: the trailing tables are GLOBAL parameters (not indexed by ids);
   * fp32 CUDA-core kernels in this round (the tensor-core formulation is round-2 work) */
  KGE_SLM = 17,     /* [ent, rel, mr1(d x k), mr2(d x k)]                    pairwise.py:525-541 */
  KGE_SME = 18,     /* [ent, rel, mu1, mu2, bu, mv1, mv2, bv] (d x d, d x 1)  pairwise.py:617-661 */
  KGE_SME_BL = 19,  /* same tables                                           pairwise.py:680-724 */
  KGE_NTN = 20,     /* [ent, rel, mr1, mr2, br(1 x k), mr(k x d*d)]          pairwise.py:919-960 */
  /* ConvKB: Conv2d(1->F,(3,w)) over the stacked [h;r;t], concat, Linear->1 with NO
   * nonlinearity in between (pointwise.py:302-318), i.e. an affine map of (h,r,t):
   *   score = <a_h,h> + <a_r,r> + <a_t,t> + c0 .
   * tables: [ent, rel, A(3 x d: rows a_h, a_r, a_t), c0(1)] with A, c0 the collapse of the
   * convolution filters with the Linear weights (host mirror: class ConvKB, pointwise.py). */
  KGE_CONVKB = 21,
  KGE_NUM_MODELS = 22
};

/* Which two operands are combined first (DESIGN.md §3.2).  TAIL: (h,r) are the
 * query side and t is the candidate — this is also the order forward() uses,
 * matching the reference's left-to-right `h + r - t` / `h*r*t`.  HEAD: (r,t)
 * are the query side and h is the candidate (Evaluator.test_head_rank,
 * pykg2vec/utils/evaluator.py:262-273). */
enum kge_grouping { KGE_GROUP_TAIL = 0, KGE_GROUP_HEAD = 1 };

typedef struct kge_model {
  int32_t model;        /* enum kge_model_id */
  int32_t dim;          /* entity embedding width d (hidden_size / ent_hidden_size) */
  int32_t rel_dim;      /* relation width (TransR rel_hidden_size); else == dim */
  int32_t l1_flag;      /* TransE-family: 1 -> L1 norm, 0 -> L2 norm (pairwise.py:73-76) */
  float margin;         /* RotatE margin (pairwise.py:791) */
  float phase_scale;    /* RotatE: (float)(pi / embedding_range) (pairwise.py:776-782) */
  int64_t num_ent;      /* rows in the entity tables passed here (a shard may pass fewer) */
  int64_t num_rel;
  const float* tables[KGE_MAX_TABLES];
} kge_model_t;

/* ---- library info ------------------------------------------------------- */
int kge_abi_version(void);
const char* kge_version(void);
const char* kge_last_error(void);

/* ---- batch scoring: replaces model.forward(h, r, t) ---------------------
 * (pykg2vec/utils/trainer.py:147-180 callers; per-model lines in kge_model_id)
 * scores[i] = f_model(tables, h[i], r[i], t[i]), i < n.  Lower = more plausible
 * for every model (the reference negates similarity models). */
int kge_score_fwd(const kge_model_t* m, int grouping, const int64_t* h, const int64_t* r,
                  const int64_t* t, int64_t n, float* scores, void* stream);

/* Backward of forward() (autograd through the ATen chain, trainer.py:298).
 * grad_tables[k] is a dense fp32 buffer shaped like tables[k] (nn.Embedding
 * dense-gradient semantics, Domain.py:8-17); row gradients are ACCUMULATED
 * into it (caller zeroes).  grad_tables[k] may be NULL to skip a table. */
int kge_score_bwd(const kge_model_t* m, const int64_t* h, const int64_t* r, const int64_t* t,
                  int64_t n, const float* grad_scores, float* const* grad_tables, void* stream);

/* Rescal.embed's side effect (pairwise.py:843-844, get_normalized_data :862-865): every row of
 * a [rows, width] table divided by its L2 norm, IN PLACE (no epsilon).  Call it on the entity
 * and relation-matrix tables before scoring, as the reference's forward() does. */
int kge_normalize_rows(float* table, int64_t rows, int64_t width, void* stream);

/* ---- losses: replace pykg2vec/utils/criterion.py ------------------------
 * Each call writes the scalar loss to loss_out[0] and, when the grad pointers
 * are non-NULL, d loss / d score (so autograd needs no second pass). */
/* Criterion.pairwise_hinge, criterion.py:26-29: sum_i max(pos_i + margin - neg_i, 0) */
int kge_loss_pairwise_hinge(const float* pos, const float* neg, int64_t n, float margin,
                            float* loss_out, float* grad_pos, float* grad_neg, void* stream);
/* Criterion.pointwise_logistic, criterion.py:32-34: mean_i softplus(target_i * preds_i) */
int kge_loss_pointwise_logistic(const float* preds, const float* target, int64_t n,
                                float* loss_out, float* grad_preds, void* stream);
/* Criterion.pariwise_logistic (sic), criterion.py:14-23: RotatE self-adversarial loss;
 * neg is [B * neg_rate] with the negatives of positive i contiguous. */
int kge_loss_selfadv(const float* pos, const float* neg, int64_t B, int32_t neg_rate, float alpha,
                     float* loss_out, float* grad_pos, float* grad_neg, void* stream);

/* get_reg() of DistMult / Complex / ComplexN3 (pointwise.py:448-458,190-202,224-238):
 * reg_out[0] = lmbda * mean_i sum_{gathered rows} sum_j g(x_j); g = x^2 (reg_type 0, "F2"),
 * x^3 signed (1, DistMult/Complex "N3"), |x|^3 (2, ComplexN3 "N3").  QuatE / OctonionE
 * (pointwise.py:696-727, :901-960) average over batch AND width: lmbda * sum_rows mean_{i,j} g(x).
 * When grad_tables is non-NULL the gradient scaled by grad_scale is accumulated into it. */
int kge_reg_fwd_bwd(const kge_model_t* m, int reg_type, float lmbda, const int64_t* h,
                    const int64_t* r, const int64_t* t, int64_t n, float* reg_out,
                    float grad_scale, float* const* grad_tables, void* stream);

/* ---- fused training step + sparse optimizer (trainer.py:147-157 + :298-299) ----
 * kge_train_pairwise_hinge_sgd: pos/neg forward + Criterion.pairwise_hinge + backward
 * + optim.SGD in two kernels.  tables_rw must alias m->tables (they are updated in
 * place); grad_scratch[k] is a ZERO-FILLED dense buffer shaped like tables[k] and is
 * zero-filled again on return.  Equivalent to optim.SGD on dense nn.Embedding
 * gradients: rows with zero gradient do not move.  loss_out[0] receives the batch
 * loss (sum over pairs).  n pairs, one negative per positive as in the reference
 * (the hinge shapes only broadcast for neg_rate == 1, criterion.py:26-29). */
int kge_train_pairwise_hinge_sgd(const kge_model_t* m, float* const* tables_rw,
                                 float* const* grad_scratch,
                                 const int64_t* pos_h, const int64_t* pos_r, const int64_t* pos_t,
                                 const int64_t* neg_h, const int64_t* neg_r, const int64_t* neg_t,
                                 int64_t n, float margin, float lr, float* loss_out, void* stream);

/* kge_train_pointwise_logistic: Trainer.train_step_pointwise (trainer.py:176-180) minus the regulariser,
 * for the pointwise row models (DistMult, Complex(N3), CP, SimplE(_ignr), ANALOGY, QuatE, OctonionE):
 * preds = model(h, r, t); loss = Criterion.pointwise_logistic(preds, y) = mean softplus(y * preds)
 * (criterion.py:32-34); backward — in ONE kernel, since d loss / d score_i depends on score_i alone.
 * y: int64 +1 / -1 labels as the generator yields them (generator.py:125-156).  loss_out[0] receives the
 * batch loss; the row gradients are ACCUMULATED into the dense grad_scratch[k] buffers (shaped like
 * tables[k]; follow with kge_reg_fwd_bwd and kge_optim_apply_rows / _dense). */
int kge_train_pointwise_logistic(const kge_model_t* m, float* const* grad_scratch, const int64_t* h,
                                 const int64_t* r, const int64_t* t, const int64_t* y, int64_t n,
                                 float* loss_out, void* stream);

/* kge_train_pairwise_selfadv: Trainer.train_step_pairwise for RotatE (trainer.py:147-157):
 * pos = model(pos triples) [B], neg = model(neg triples) [B * neg_rate] (the negatives of positive i are
 * neg[i*neg_rate .. (i+1)*neg_rate), generator.py:94-121), loss = Criterion.pariwise_logistic(pos, neg,
 * neg_rate, alpha) — the self-adversarial loss, criterion.py:14-23, softmax weights detached — and backward, in
 * ONE kernel (a warp owns a positive with its negatives).  loss_out[0] receives the batch loss (the same bits
 * as kge_loss_selfadv on the same scores); the row gradients are ACCUMULATED into grad_scratch[k].
 * KGE_ENOTSUP for other models, and when neg_rate needs more shared memory than a CTA has (then use
 * kge_score_fwd + kge_loss_selfadv + kge_score_bwd). */
int kge_train_pairwise_selfadv(const kge_model_t* m, float* const* grad_scratch, const int64_t* pos_h,
                               const int64_t* pos_r, const int64_t* pos_t, const int64_t* neg_h,
                               const int64_t* neg_r, const int64_t* neg_t, int64_t B, int32_t neg_rate,
                               float alpha, float* loss_out, void* stream);

/* Sparse optimizer.step() for the rows touched by the triples (h[i], r[i], t[i]):
 * takes the accumulated row gradients out of grad_scratch (as filled by
 * kge_score_bwd / kge_reg_fwd_bwd; left zero-filled) and applies
 *   optimizer 0: torch.optim.SGD      w -= lr * g                     (trainer.py:117-121)
 *   optimizer 1: torch.optim.Adagrad  s += g*g; w -= lr*g/(sqrt(s)+eps) (trainer.py:122-126)
 * state[k] (Adagrad) is shaped like tables[k].  For both optimizers rows with zero
 * gradient are left untouched by the dense reference optimizers too, so the result
 * equals the dense step. */
int kge_optim_apply_rows(const kge_model_t* m, float* const* tables_rw, float* const* grad_scratch,
                         float* const* state, int optimizer, const int64_t* h, const int64_t* r,
                         const int64_t* t, int64_t n, float lr, float eps, void* stream);

/* Dense optimizer.step() for ONE parameter tensor of n floats (any shape): the accumulated gradient is
 * taken out of `grad` (a dense buffer filled by kge_score_bwd / kge_reg_fwd_bwd / an all-reduce of such
 * buffers; left zero-filled) and applied in place to w.
 *   optimizer 0: torch.optim.SGD; 1: torch.optim.Adagrad (state1 = sum of squares, eps 1e-10);
 *   optimizer 2: torch.optim.Adam — the reference's default `-opt adam` (pykg2vec/common.py:50,
 *   utils/trainer.py:112-116): state1 = exp_avg, state2 = exp_avg_sq, step = 1-based step count,
 *   torch's update order (lerp, mul+addcmul, sqrt / sqrt(bias_correction2) + eps, addcdiv).  Dense Adam
 *   moves every element every step (moments of gradient-free rows keep decaying), so this is one
 *   HBM-bound sweep over the tensor, not a sparse row update; results equal torch's to rounding.
 * Used by the fused training steps with -opt adam and by data-parallel training after the gradient
 * all-reduce (pykg2vec_b200/sharding.py).  Tensors must be 16-byte aligned. */
int kge_optim_apply_dense(float* w, float* grad, float* state1, float* state2, int64_t n, int optimizer,
                          float lr, float eps, float beta1, float beta2, int64_t step, void* stream);

/* ---- 1-vs-all link-prediction ranks: replaces Evaluator.test ------------
 * (pykg2vec/utils/evaluator.py:309-334 + MetricCalculator.get_*_rank :70-123)
 *
 * For query i = (qh[i], qr[i], qt[i]) and candidate entity rows
 * [row_lo, row_hi) of the tables in `m` (m->num_ent == row_hi - row_lo rows are
 * addressable, local row k is global entity row_lo + k):
 *   counts[i*4+0] += #{e : score(qh,qr,e) <  score(qh,qr,qt)}            (tail, raw)
 *   counts[i*4+1] += the same minus #{e in filt_t[i], e != qt : ...}      (tail, filtered)
 *   counts[i*4+2], counts[i*4+3]: likewise for heads with filt_h (tr_h).
 * i.e. the 0-based ranks MetricCalculator computes when scores are tie-free.
 * Query-side rows are read from `mq` (normally == m; for a row-sharded table a
 * compact table of gathered query rows with qh/qt re-indexed into it, while
 * tgt_h/tgt_t keep GLOBAL entity ids used only for id comparisons and filters).
 * Filters are CSR over queries with GLOBAL entity ids (hr_t / tr_h of
 * pykg2vec/data/kgcontroller.py:410-428): ptr[Q+1], idx[nnz]; nnz is passed
 * explicitly (it lives in device memory as ptr[Q]).  Pointers may be NULL /
 * nnz 0 (then filtered == raw).  Q <= 65535 per call (batch larger test sets).
 * counts is ACCUMULATED (caller zeroes), int32 [Q,4]; partial counts of
 * different row shards add up to the global rank (one all-reduce).
 * workspace: >= kge_rank_workspace_bytes(m, Q) bytes of device memory. */
int64_t kge_rank_workspace_bytes(const kge_model_t* m, int64_t Q);
int kge_rank_1vsall(const kge_model_t* m, const kge_model_t* mq, int64_t row_lo, int64_t row_hi,
                    const int64_t* qh, const int64_t* qr, const int64_t* qt,
                    const int64_t* tgt_h, const int64_t* tgt_t, int64_t Q,
                    const int64_t* filt_t_ptr, const int64_t* filt_t_idx, int64_t filt_t_nnz,
                    const int64_t* filt_h_ptr, const int64_t* filt_h_idx, int64_t filt_h_nnz,
                    int32_t* counts, void* workspace, int64_t workspace_bytes, int flags,
                    void* stream);
/* flags for kge_rank_1vsall */
#define KGE_RANK_FORCE_GATHER 1 /* use the untiled gather sweep even where a tiled kernel exists */
#define KGE_RANK_TAIL_ONLY 2
#define KGE_RANK_HEAD_ONLY 4
#define KGE_RANK_SINGLE_STREAM 8 /* do not overlap the two directions on an internal side stream */
#define KGE_RANK_NO_TC 16 /* keep the sweep on the fp32 pipe (no tensor-core level; same counts either way) */
#define KGE_RANK_PROFILE 32 /* record CUDA events around each direction's main sweep kernel, see kge_rank_last_sweep_ms */

/* Measurement aid (bench.py's roofline entry): after a kge_rank_1vsall call with KGE_RANK_PROFILE from the
 * same host thread, *ms receives the device time of direction 0 (tail) / 1 (head)'s main sweep kernel —
 * tc_sweep_kernel, or sweep_tiled_kernel with KGE_RANK_NO_TC — measured by CUDA events recorded around
 * that launch on the stream it ran on (waits for the kernel).  Not usable inside a graph capture.
 * A full rank call of a tensor-core model sweeps BOTH directions in one launch: it is reported as direction 0,
 * kge_rank_last_sweep_directions() returns 2 (1 for per-direction launches, 0 when nothing was profiled) and
 * direction 1 has no launch of its own (KGE_EINVAL). */
int kge_rank_last_sweep_ms(int direction, float* ms);
int kge_rank_last_sweep_directions(void);
/* Measurement aid: per-role clock64 timeline of CTA (0,0) of subsequent tc_sweep_kernel launches into the
 * device buffer buf[3][64] (NULL = off): role 0 TMA producer, 1 consumer warpgroup start, 2 epilogue begin / end
 * per tile, slot 63 of role 2 the kernel entry (see kge_rank.cu);
 * behind them buf[192 + 2 i], buf[193 + 2 i] = %globaltimer (ns) at entry / exit of CTA i (linear id < 1024),
 * and buf[2*64 + 62] = clock64 at the exit of CTA 0: the buffer must hold 192 + 2048 int64. */
int kge_debug_set_tc_trace(long long* buf);

/* Two-level exact sweep (TransE -l1 False, DistMult, CP, ComplEx, RESCAL, RotatE; >= 1024 candidate rows):
 * level 1 evaluates the Q x N x K contraction on the tensor cores (wgmma, bf16 x 3 split, fp32
 * accumulation in registers) and counts every candidate whose accumulator clears the query's threshold by
 * more than a proven error bound of that (query, candidate) pair; level 2 re-evaluates the few (query, candidate) pairs inside the
 * band in the canonical fp32 arithmetic.  The counts equal the fp32 specification's for every input
 * (DESIGN.md §4b).  kge_rank_tc_probe exposes level 1 of ONE direction (0 tail, 1 head) for tests and
 * measurements: dots[Q * (row_hi-row_lo)] receives the raw accumulators D(q, c) (may be NULL);
 * tau[Q*4 + (row_hi-row_lo)] (may be NULL) the band: per query (centre, a, b, e), then per candidate its norm
 * bound n_c — half(q,c) = a + b n_c + e n_c^2; certainly better: D - centre > half; certainly not:
 * D - centre < -half; otherwise the pair is resolved exactly;
 * counts[Q*4] is accumulated exactly as by kge_rank_1vsall (raw and "filtered" columns both get the raw
 * count: no filter pass here).  KGE_ENOTSUP when the model / table size has no tensor-core sweep. */
int kge_rank_tc_probe(const kge_model_t* m, const kge_model_t* mq, int64_t row_lo, int64_t row_hi,
                      const int64_t* qh, const int64_t* qr, const int64_t* qt, int64_t Q, int direction,
                      float* dots, float* tau, int32_t* counts, void* workspace, int64_t workspace_bytes,
                      void* stream);

/* ---- per-relation entity projection (relation-grouped evaluation of TransH / TransD) ----------
 * TransH.embed/_projection (pykg2vec/models/pairwise.py:166-182) and TransD.embed/_projection
 * (:240-249,275-278) project the h and t rows with a vector chosen by the relation and then apply
 * TransE's distance.  For a fixed relation r this writes the projected row of EVERY entity,
 *   KGE_TRANSH: out[e] = ent[e] - (ent[e] . w~_r) w~_r,  w~_r = w[r] / max(|w[r]|, 1e-12)
 *   KGE_TRANSD: out[e] = ent[e] + (ent[e] . ent_map[e]) rel_map[r]
 * in exactly the arithmetic kge_score_fwd applies to the rows of a triple, so that
 *   score_model(h, r, t) == score_TransE over tables [out, rel] at (h, r, t)   bit for bit
 * and the test triples of relation r can be ranked by kge_rank_1vsall with a KGE_TRANSE model over
 * [out, rel] (the tiled sweep) instead of the per-pair gather sweep.  out: [num_ent, dim] fp32. */
int kge_project_entities(const kge_model_t* m, int64_t r, float* out, void* stream);

/* KGE_TRANSR is accepted as well: out[e] = normalize(ent[e]) . M_r, [num_ent, rel_dim]
 * (TransR.transform on the normalised rows, pairwise.py:405-413,430-442).  Together with the ONCE
 * normalised relation rows written by kge_normalize_rows_to (F.normalize(rel), pairwise.py:430-432, in
 * the canonical arithmetic: row * (1 / max(|row|, 1e-12))), TransE of width rel_dim over
 * [out, normalised rel] applies the reference's second normalisation (:463-465) and reproduces
 * score_TransR bit for bit.  (Proved on the oracle with the emulated kernels, tests/test_emu_project.py;
 * the relation-grouped Evaluator uses it for TransR only on request — not timed.) */
int kge_normalize_rows_to(const float* table, int64_t rows, int64_t width, float* out, void* stream);

/* ---- projection-model tail: x.E^T + b -> sigmoid, multi-class BCE, rank counts ----------
 * The last layer shared by the reference's projection models:
 *   ConvE.inner_forward    pykg2vec/models/projection.py:100-102   (torch.matmul(x, E.T); + b; sigmoid)
 *   TuckER :335-336, InteractE :444-447, HypER :607-609, AcrE :735-738; ProjE_pointwise.g :248-256 (no bias)
 * x [B,k] is the trunk's output (device, fp32 row-major), ent the [N,k] entity table, bias [N] or NULL.
 * preds[b*N + n] = sigmoid(sum_j x[b,j] ent[n,j] + bias[n]); canonical arithmetic: one sequential
 * fma chain over j from 0, one add, canonical sigmoid (DESIGN.md §3 rule 8) — bit-identical to
 * oracle/kge_oracle.c and to what kge_proj_rank compares, whatever CTA tile the launcher picks
 * (64x64 / 64x128 / 128x128 by problem size; the environment variable KGE_PROJ_TILE=0|1|2 forces one —
 * a testing / benchmarking aid, read at every call). */
int kge_proj_tail_fwd(const float* x, const float* ent, const float* bias, int64_t B, int64_t N,
                      int32_t k, float* preds, void* stream);

/* Backward of kge_proj_tail_fwd (autograd through matmul/add/sigmoid, trainer.py:298).  With
 * g = grad_preds * preds * (1 - preds):  grad_x[B,k] += g E;  grad_ent[N,k] += g^T x;
 * grad_bias[N] += column sums of g.  All three are ACCUMULATED (caller zeroes; grad_ent is the dense
 * nn.Embedding gradient the gather of the input rows also adds into) and may be NULL. */
int kge_proj_tail_bwd(const float* grad_preds, const float* preds, const float* x, const float* ent,
                      int64_t B, int64_t N, int32_t k, float* grad_x, float* grad_ent,
                      float* grad_bias, void* stream);

/* One direction of Criterion.multi_class_bce (pykg2vec/utils/criterion.py:41-50):
 *   y = labels * label_scale + label_shift       (:43-45: scale = 1 - label_smoothing, shift = 1/tot_entity;
 *                                                 pass 1, 0 when label_smoothing is None)
 *   loss_out[0] = mean_{b,n} BCEWithLogits(preds, y)   (:46-47, applied to the already-sigmoided preds
 *                                                 exactly as the reference does)
 * and, when grad_preds is non-NULL, grad_preds = grad_scale * d loss / d preds.  labels is the dense
 * [B,N] fp32 matrix the reference's generator yields (generator.py:160-230). */
int kge_proj_bce(const float* preds, const float* labels, int64_t B, int64_t N, float label_scale,
                 float label_shift, float grad_scale, float* loss_out, float* grad_preds, void* stream);

/* The dense label matrices of a PROJECTION_BASED batch, built on the device: what
 * process_function_multiclass (pykg2vec/data/generator.py:160-236) assembles on the host per batch with
 * torch.sparse(...).to_dense() and ships as two [B, N] float tensors.  labels[b, :] = 0 except 1.0 at the
 * entities idx[ptr[row] .. ptr[row+1]) with row = rows[b] (rows == NULL: row = b).  ptr/idx are a CSR of
 * hr_t_train (or tr_h_train) over its distinct keys, rows[b] the key row of training triple b — so a
 * batch moves B ids instead of B*N floats over PCIe.  The -1 entries the reference adds when neg_rate > 0
 * (ProjE only) come from kge_proj_labels_negatives, called after this. */
int kge_proj_labels(const int64_t* rows, const int64_t* ptr, const int64_t* idx, int64_t B, int64_t N,
                    float* labels, void* stream);

/* The -1 labels of process_function_multiclass with neg_rate > 0 (pykg2vec/data/generator.py:200-238, used by
 * ProjE_pointwise): one permutation of the entities per batch, and its first min(100, N) ids are negatives of
 * every row and both directions unless they are positives of that row.  After kge_proj_labels:
 *   labels[b, neg[j]] = -1 for b < B, j < n_neg, wherever labels[b, neg[j]] == 0.
 * neg: n_neg DISTINCT entity ids (device int64).  B = 0 or n_neg = 0 is a no-op. */
int kge_proj_labels_negatives(float* labels, int64_t B, int64_t N, const int64_t* neg, int64_t n_neg, void* stream);

/* predict_tail_rank / predict_head_rank (projection.py:119-125: topk of -preds over all N entities,
 * one query at a time) + MetricCalculator.get_*_rank (evaluator.py:70-123), for Q queries at once and
 * without materialising the [Q,N] prediction matrix:
 *   counts[q*4 + 2*direction]     += #{n : pred(q,n) > pred(q,tgt[q])}
 *   counts[q*4 + 2*direction + 1] += the same minus #{n in filter row q, n != tgt[q] : ...}
 * direction 0 = tail (x from (h, r), tgt = t, filter hr_t), 1 = head (x from (t, r + R), tgt = h, tr_h).
 * Filters: CSR over queries, ptr[Q+1] / idx[nnz] int64 (NULL / nnz 0 -> filtered == raw).
 * workspace >= kge_proj_rank_workspace_bytes(Q) bytes of device memory. */
int64_t kge_proj_rank_workspace_bytes(int64_t Q);
int kge_proj_rank(const float* x, const float* ent, const float* bias, int64_t Q, int64_t N, int32_t k,
                  const int64_t* tgt, const int64_t* filt_ptr, const int64_t* filt_idx, int64_t filt_nnz,
                  int32_t direction, int32_t* counts, void* workspace, int64_t workspace_bytes,
                  void* stream);

/* ---- ConvE trunk, inference mode ----------------------------------------------------------
 * ConvE.forward + inner_forward up to the x.E^T product (pykg2vec/models/projection.py:104-112,
 * :86-99) with self.training == False: x[q,:] = relu(fc(flatten(relu(bn1(conv2d_1(bn0(
 * [ent[e[q]] ; rel[r[q]]] viewed as [1, 2*hidden_size_2, hidden_size_1])))))))  — dropouts are
 * identities, BatchNorm uses running statistics, bn2 is not applied (projection.py:97-98).
 * All pointers are device fp32 tensors with the reference's state_dict shapes:
 *   ent [N,k], rel [2R,k] (reciprocal relations: the head direction passes r + R, :107-108),
 *   bn0_* [1], conv_weight [32,1,3,3], conv_bias [32], bn1_* [32], fc_weight [k, F], fc_bias [k],
 *   F = 32 * (2*hidden_size_2 - 2) * (hidden_size_1 - 2), hidden_size_2 = hidden_size / hidden_size_1.
 * x is [Q,k]; workspace >= kge_conve_trunk_workspace_bytes() bytes (the flattened feature maps).
 * Training (batch statistics, dropout, autograd): kge_conve_train_* below. */
typedef struct kge_conve {
  int32_t hidden_size, hidden_size_1;
  float bn0_eps, bn1_eps;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* bn0_mean; const float* bn0_var;
  const float* conv_weight; const float* conv_bias;
  const float* bn1_weight; const float* bn1_bias; const float* bn1_mean; const float* bn1_var;
  const float* fc_weight; const float* fc_bias;
} kge_conve_t;
int64_t kge_conve_trunk_workspace_bytes(const kge_conve_t* p, int64_t Q);
int kge_conve_trunk_fwd(const kge_conve_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                        void* workspace, int64_t workspace_bytes, void* stream);

/* ---- ConvE trunk, training mode ------------------------------------------------------------
 * ConvE.inner_forward up to the x.E^T product (pykg2vec/models/projection.py:86-99) with self.training == True,
 * forward and backward; replaces the reference's torch layers bn0 -> inp_drop -> conv2d_1 -> bn1 -> relu ->
 * feat_drop -> fc -> hidden_drop -> bn2 -> relu and their autograd.  The Q = G * B rows are G groups of B rows
 * (G = 2: the tail and head forwards of train_step_projection, trainer.py:159-174, as one call); every BatchNorm
 * uses the batch statistics of its own group, and the running statistics are updated group after group exactly
 * as G sequential nn.BatchNorm calls do (momentum from the struct, unbiased variance n / (n - 1));
 * num_batches_tracked is the caller's.  Running-statistic pointers: all six set, or all NULL (no update).
 * Dropout is explicit noise, bernoulli(1 - p) / (1 - p) as torch draws it (each may be NULL = no dropout):
 *   noise0 [Q, 2k] (inp_drop), noise1 [Q, 32] (feat_drop, Dropout2d: one value per channel), noise2 [Q, k].
 * Images: as kge_conve_trunk_fwd (2k <= 4096, hidden_size_1 >= 3, hidden_size_2 >= 2; KGE_ENOTSUP beyond);
 * B >= 2 (a one-row BatchNorm1d raises in the reference) and Q a multiple of B, else KGE_EINVAL.
 *
 * kge_conve_train_fwd: x [Q, k].  Every statistic is reduced in a fixed order that does not depend on the grid
 * (DESIGN.md §3, ConvE training), so x and the running statistics are bit-reproducible.  The workspace
 * (kge_conve_train_workspace_bytes(p, Q, B) bytes) keeps what the backward reads: pass the same workspace, unmodified,
 * to kge_conve_train_bwd.
 * kge_conve_train_bwd: from gx = d loss / d x [Q, k] (kge_proj_tail_bwd's grad_x) and the forward's x, ACCUMULATES
 * into KGE_CONVE_TRAIN_GRADS dense buffers shaped like the parameters (caller zeroes; none may be NULL), in
 * ConvE.parameters() order without the tail's bias row: ent, rel, bn0.weight, bn0.bias, conv2d_1.weight,
 * conv2d_1.bias, bn1.weight, bn1.bias, fc.weight, fc.bias, bn2.weight, bn2.bias.  The entity / relation rows are
 * scattered with float atomics (ids repeat); every other sum runs in a fixed order.  No entry point allocates. */
#define KGE_CONVE_TRAIN_GRADS 12
typedef struct kge_conve_train {
  int32_t hidden_size, hidden_size_1;
  float bn0_eps, bn1_eps, bn2_eps;
  float bn0_momentum, bn1_momentum, bn2_momentum;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* conv_weight; const float* conv_bias;
  const float* bn1_weight; const float* bn1_bias; const float* fc_weight; const float* fc_bias;
  const float* bn2_weight; const float* bn2_bias;
  float* bn0_mean; float* bn0_var; float* bn1_mean; float* bn1_var; float* bn2_mean; float* bn2_var;
} kge_conve_train_t;
int64_t kge_conve_train_workspace_bytes(const kge_conve_train_t* p, int64_t Q, int64_t B);
int kge_conve_train_fwd(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* noise0, const float* noise1, const float* noise2, float* x, void* workspace,
                        int64_t workspace_bytes, void* stream);
int kge_conve_train_bwd(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* noise0, const float* noise1, const float* noise2, const float* gx,
                        const float* x, float* const* grads, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- HypER trunk, inference mode -----------------------------------------------------------
 * HypER.forward up to the x.E^T product (pykg2vec/models/projection.py:581-606) with
 * self.training == False: dropouts are identities and bn0 / bn1 / bn2 use their running statistics.
 * Per query q (one relation-generated filter bank per query, a hypernetwork):
 *   v = bn0(ent[e[q]])                                  [de]
 *   w = fc1(rel[r[q]]) viewed [32][9]                   channel c uses w[9c .. 9c+8]
 *   f[c][j] = bn1_c(sum_{t<9} w[c][t] * v[j+t])          j < de-8; no conv bias, no ReLU
 *   x[q,:] = relu(bn2(fc(f flattened channel-major)))
 * `direction` does not enter: the head direction passes (t, r) (no reciprocal relations).
 * All pointers are device fp32 tensors with the reference's state_dict shapes:
 *   ent [N,de], rel [num_rel,dr], bn0_* [1], fc1_weight [288,dr], fc1_bias [288], bn1_* [32],
 *   fc_weight [de, F], fc_bias [de], bn2_* [de], F = 32 * (de - 8).
 * The filters of all num_rel relations are computed on every call (one GEMM of num_rel x 288 x dr).
 * x is [Q,de]; workspace >= kge_hyper_trunk_workspace_bytes() bytes (filter table, flattened
 * feature maps and the Linear layer's slice partials).  Q = 0 is a no-op (e, r and x may then be NULL).
 * KGE_ENOTSUP when de < 9 or the entity row does not fit the feature kernel's shared memory (de > 4096). */
typedef struct kge_hyper {
  int32_t ent_hidden_size, rel_hidden_size;
  int64_t num_rel;
  float bn0_eps, bn1_eps, bn2_eps;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* bn0_mean; const float* bn0_var;
  const float* fc1_weight; const float* fc1_bias;
  const float* bn1_weight; const float* bn1_bias; const float* bn1_mean; const float* bn1_var;
  const float* fc_weight; const float* fc_bias;
  const float* bn2_weight; const float* bn2_bias; const float* bn2_mean; const float* bn2_var;
} kge_hyper_t;
int64_t kge_hyper_trunk_workspace_bytes(const kge_hyper_t* p, int64_t Q);
int kge_hyper_trunk_fwd(const kge_hyper_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                        void* workspace, int64_t workspace_bytes, void* stream);

/* ---- HypER trunk, training mode ------------------------------------------------------------
 * HypER.forward up to the x.E^T product (pykg2vec/models/projection.py:581-606) with self.training == True, forward
 * and backward; replaces the reference's torch layers bn0 -> inp_drop -> fc1 -> grouped conv -> bn1 ->
 * feature_map_drop -> fc -> hidden_drop -> bn2 -> relu and their autograd.  Per query q (no ReLU after bn1):
 *   w = fc1(rel[r[q]]) [32][9];  v = bn0(ent[e[q]]) * noise0;  z1[c][j] = sum_{t<9} w[c][t] v[j+t] (j < de-8);
 *   x[q,:] = relu(bn2((fc(flatten(bn1(z1) * noise1)) * noise2)))
 * The Q = G * B rows are G groups of B rows (G = 2: the tail and head forwards of train_step_projection as one call);
 * every BatchNorm uses the batch statistics of its own group, and the running statistics are updated group after
 * group as G sequential nn.BatchNorm calls do (momentum from the struct, unbiased variance); num_batches_tracked is
 * the caller's.  Running-statistic pointers: all six set, or all NULL (no update).  A filter has the same bits as
 * kge_hyper_trunk_fwd's filter of that relation.
 * Dropout is explicit noise, bernoulli(1 - p) / (1 - p) as torch draws it (each may be NULL = no dropout):
 *   noise0 [Q, de] (inp_drop), noise1 [Q, 32] (feature_map_drop, Dropout2d: one value per channel), noise2 [Q, de].
 * ent_padding_idx / rel_padding_idx: the embeddings' padding_idx (-1: none); that row receives no lookup gradient
 * (nn.Embedding's rule), its value is read as any other.
 * Widths: 9 <= de <= 4096 (KGE_ENOTSUP beyond, as kge_hyper_trunk_fwd); B >= 2 (a one-row BatchNorm1d raises in the
 * reference) and Q a multiple of B, else KGE_EINVAL.
 *
 * kge_hyper_train_fwd: x [Q, de].  Every statistic is reduced in a fixed order that does not depend on the grid, so x
 * and the running statistics are bit-reproducible.  The workspace (kge_hyper_train_workspace_bytes(p, Q, B) bytes)
 * keeps what the backward reads: pass the same workspace, unmodified, to kge_hyper_train_bwd.
 * kge_hyper_train_bwd: from gx = d loss / d x [Q, de] and the forward's x, ACCUMULATES into KGE_HYPER_TRAIN_GRADS dense
 * buffers shaped like the parameters (caller zeroes; none may be NULL), in this order: ent, rel, bn0.weight,
 * bn0.bias, bn1.weight, bn1.bias, fc.weight, fc.bias, bn2.weight, bn2.bias, fc1.weight, fc1.bias.  The entity /
 * relation rows are scattered with float atomics (ids repeat); every other sum runs in a fixed order.  No entry point
 * allocates. */
#define KGE_HYPER_TRAIN_GRADS 12
typedef struct kge_hyper_train {
  int32_t ent_hidden_size, rel_hidden_size;
  int64_t ent_padding_idx, rel_padding_idx;
  float bn0_eps, bn1_eps, bn2_eps;
  float bn0_momentum, bn1_momentum, bn2_momentum;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* bn1_weight; const float* bn1_bias;
  const float* fc_weight; const float* fc_bias; const float* bn2_weight; const float* bn2_bias;
  const float* fc1_weight; const float* fc1_bias;
  float* bn0_mean; float* bn0_var; float* bn1_mean; float* bn1_var; float* bn2_mean; float* bn2_var;
} kge_hyper_train_t;
int64_t kge_hyper_train_workspace_bytes(const kge_hyper_train_t* p, int64_t Q, int64_t B);
int kge_hyper_train_fwd(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* noise0, const float* noise1, const float* noise2, float* x, void* workspace,
                        int64_t workspace_bytes, void* stream);
int kge_hyper_train_bwd(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* noise0, const float* noise1, const float* noise2, const float* gx,
                        const float* x, float* const* grads, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- InteractE trunk, inference mode -------------------------------------------------------
 * InteractE.forward up to the x.E^T product (pykg2vec/models/projection.py:425-442) with
 * self.training == False: dropouts are identities and bn0 / bn1 / bn2 use their running statistics.
 * P = feature_permutation, F = num_filters, ks = kernel_size, H = 2*reshape_width image rows,
 * W = reshape_height image columns, k = reshape_width*reshape_height, pad = ks/2.  Per query q:
 *   comb = [ent[e[q]] ; rel[r[q]]]                                  [2k]
 *   img[p][i][j] = bn0_p(comb[perm[p][i*W + j]])                    P chequer-permuted images [H][W]
 *   f[p*F+f][i][j] = relu(bn1_{p*F+f}(sum_{u,v<ks} conv_filt[f][u][v] * img[p][(i+u-pad) mod H][(j+v-pad) mod W]))
 *   x[q,:] = relu(bn2(fc(f flattened channel-major)))
 * (circular padding, filter f on every image, no conv bias).  `direction` does not enter: the head direction
 * passes (t, r) (no reciprocal relations).  perm is the model's chequer permutation, int64 [P, 2k] on the device.
 * The other pointers are device fp32 tensors with the reference's state_dict shapes:
 *   ent [N,k], rel [num_rel,k], bn0_* [P], conv_filt [F,1,ks,ks], bn1_* [P*F], fc_weight [k, P*F*H*W],
 *   fc_bias [k], bn2_* [k].
 * x is [Q,k]; workspace >= kge_interacte_trunk_workspace_bytes() bytes (the flattened feature maps and the
 * Linear layer's slice partials, ~(P*F*H*W + ceil(P*F*H*W / 512) * k) floats per query, 214 KB at the default
 * (1, 96, 9, 20x10) shape: callers bound it by splitting Q).  Q = 0 is a no-op (e, r and x may then be NULL).
 * KGE_ENOTSUP for an even ks or ks < 3 (the reference's forward fails there), pad > min(H, W), or when the
 * filter bank (ks*ks*ceil8(F) floats), the bn1 folds (2*P*ceil8(F)) and the P padded images
 * ((H+2pad)*(W+2pad) each) exceed 227 KB, the per-block shared memory of sm_90. */
typedef struct kge_interacte {
  int32_t feature_permutation, num_filters, kernel_size, reshape_height, reshape_width;
  int64_t num_rel;
  float bn0_eps, bn1_eps, bn2_eps;
  const int64_t* perm;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* bn0_mean; const float* bn0_var;
  const float* conv_filt;
  const float* bn1_weight; const float* bn1_bias; const float* bn1_mean; const float* bn1_var;
  const float* fc_weight; const float* fc_bias;
  const float* bn2_weight; const float* bn2_bias; const float* bn2_mean; const float* bn2_var;
} kge_interacte_t;
int64_t kge_interacte_trunk_workspace_bytes(const kge_interacte_t* p, int64_t Q);
int kge_interacte_trunk_fwd(const kge_interacte_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                            void* workspace, int64_t workspace_bytes, void* stream);

/* ---- InteractE trunk, training mode ---------------------------------------------------------
 * InteractE.forward up to the x.E^T product (pykg2vec/models/projection.py:425-442) with self.training == True,
 * forward and backward; replaces the reference's torch layers bn0 -> inp_drop -> circular conv -> bn1 -> relu ->
 * feature_map_drop -> fc -> hidden_drop -> bn2 -> relu and their autograd.  Geometry and per-query function as
 * kge_interacte_trunk_fwd (H = 2*reshape_width, W = reshape_height, HW = H*W = 2k, pad = ks/2, C1 = P*F):
 *   img[p] = comb[perm[p]] viewed [H][W];  v[p] = bn0_p(img[p]) * noise0[q, p, :, :]
 *   z1[p*F+f][i][j] = sum_{u,v<ks} conv_filt[f][u][v] * v[p][(i+u-pad) mod H][(j+v-pad) mod W]   (no bias)
 *   x[q,:] = relu(bn2((fc(flatten(relu(bn1(z1)) * noise1[q, c]))) * noise2[q, :]))
 * The Q = G * B rows are G groups of B rows (G = 2: the tail and head forwards of train_step_projection as one call);
 * every BatchNorm uses the batch statistics of its own group (bn0 per image channel p over B*HW values, bn1 per
 * channel over B*HW, bn2 per feature over B), and the running statistics are updated group after group as G
 * sequential nn.BatchNorm calls do (momentum from the struct, unbiased variance); num_batches_tracked is the
 * caller's.  Running-statistic pointers: all six set, or all NULL (no update).  perm: int64 [P, 2k] on the device,
 * every row a permutation of 0 .. 2k-1 (the backward's un-permute relies on it; not checked here).
 * Dropout is explicit noise, bernoulli(1 - p) / (1 - p) as torch draws it (each may be NULL = no dropout):
 *   noise0 [Q, P*2k] (inp_drop on [Q, P, H, W]), noise1 [Q, C1] (feature_map_drop, Dropout2d: one value per
 *   channel), noise2 [Q, k] (hidden_drop).  The embeddings have no padding_idx.
 * Shapes: the bounds of kge_interacte_trunk_fwd (odd ks >= 3, pad <= min(H, W), filter bank + bn1 folds + P padded
 * images within 227 KB of shared memory; KGE_ENOTSUP beyond); B >= 2 (a one-row BatchNorm1d raises in the reference)
 * and Q a multiple of B, else KGE_EINVAL.
 *
 * kge_interacte_train_fwd: x [Q, k].  Every statistic is reduced in a fixed order that does not depend on the grid,
 * so x and the running statistics are bit-reproducible.  The workspace (kge_interacte_train_workspace_bytes(p, Q, B)
 * bytes) keeps what the backward reads: pass the same workspace, unmodified, to kge_interacte_train_bwd, once (the
 * backward overwrites the forward's feature maps with their gradient).  It holds two [Q, P*F*H*W] arrays (z1 and
 * feat / d feat), the Linear layer's slice partials [ceil(P*F*H*W / 512), Q, k], the per-query d conv_filt
 * [Q, F*ks*ks] and O(Q * (P*HW + k)) more: ~103 MB at (1, 96, 9, 20x10) with Q = 256, ~250 MB at (4, 64, 7).  The
 * statistics span the group, so the call cannot be split over Q.
 * kge_interacte_train_bwd: from gx = d loss / d x [Q, k] and the forward's x, ACCUMULATES into
 * KGE_INTERACTE_TRAIN_GRADS dense buffers shaped like the parameters (caller zeroes; none may be NULL), in this order:
 * ent, rel, bn0.weight, bn0.bias, conv_filt, bn1.weight, bn1.bias, fc.weight, fc.bias, bn2.weight, bn2.bias.  The
 * entity / relation rows are scattered with float atomics (ids repeat); every other sum runs in a fixed order.  No
 * entry point allocates. */
#define KGE_INTERACTE_TRAIN_GRADS 11
typedef struct kge_interacte_train {
  int32_t feature_permutation, num_filters, kernel_size, reshape_height, reshape_width;
  float bn0_eps, bn1_eps, bn2_eps;
  float bn0_momentum, bn1_momentum, bn2_momentum;
  const int64_t* perm;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* conv_filt;
  const float* bn1_weight; const float* bn1_bias; const float* fc_weight; const float* fc_bias;
  const float* bn2_weight; const float* bn2_bias;
  float* bn0_mean; float* bn0_var; float* bn1_mean; float* bn1_var; float* bn2_mean; float* bn2_var;
} kge_interacte_train_t;
int64_t kge_interacte_train_workspace_bytes(const kge_interacte_train_t* p, int64_t Q, int64_t B);
int kge_interacte_train_fwd(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                            const float* noise0, const float* noise1, const float* noise2, float* x, void* workspace,
                            int64_t workspace_bytes, void* stream);
int kge_interacte_train_bwd(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                            const float* noise0, const float* noise1, const float* noise2, const float* gx,
                            const float* x, float* const* grads, void* workspace, int64_t workspace_bytes,
                            void* stream);

/* ---- AcrE trunk, inference mode ------------------------------------------------------------
 * AcrE.forward up to the x.E^T product (pykg2vec/models/projection.py:706-734) with self.training == False:
 * dropouts are identities and bn0 / bn1 / bn2 use their running statistics.  C = in_channels, conv l is a
 * 3x3 conv with stride 1 and padding = dilation = its atrous rate (zero padding: the maps stay 20 x 20).
 * Per query q:
 *   img[20][20] = bn0([ent[e[q]] ; rel[r[q]]])                      the two 200-wide rows, 10 x 20 each
 *   serial (way 0):   y = conv3(conv2(conv1(img))) + img            1 -> C -> C -> C, img on every channel
 *   parallel (way 1): y[c] = W_gate_e([img ; conv1(img)[c] ; conv2(img)[c] ; conv3(img)[c]])   each conv 1 -> C
 *   x[q,:] = relu(bn2(fc(relu(bn1(y)) flattened channel-major)))
 * `direction` does not enter: rel is indexed with r as given (rows num_rel/2.. of the reference's [2R, k] table
 * are never read) and the head direction passes (t, r).  Pointers are device fp32 tensors with the reference's
 * state_dict shapes: ent [N,200], rel [num_rel,200], bn0_* [1], conv1_weight [C,1,3,3], conv2/3_weight
 * [C,C,3,3] (serial) or [C,1,3,3] (parallel), conv*_bias [C] — all three NULL for acre_bias = False, W_gate_e
 * weight [400,1600] and bias [400] (parallel only; ignored by the serial way), bn1_* [C], fc_weight
 * [200, C*400], fc_bias [200], bn2_* [200].
 * x is [Q,200]; workspace >= kge_acre_trunk_workspace_bytes() bytes: per query the gate input (parallel only,
 * C*1600 floats, 205 KB at C = 32), the features (C*400 floats, 51 KB at C = 32) and the Linear layer's slice
 * partials (ceil(C*400/512)*200 floats); callers bound it by splitting Q.  Q = 0 is a no-op (e, r and x may
 * then be NULL).
 * KGE_EINVAL: way not 0 / 1, an atrous rate < 1, in_channels < 1, num_rel < 1, one or two (not zero or three)
 * NULL conv biases, a NULL required pointer, or Q beyond one call's grid.  KGE_ENOTSUP: hidden_size != 200 (the
 * reference's 10 x 20 view), a serial C whose maps and weight bank exceed 227 KB of shared memory
 * (4*(400 + 800*C + 9*C*ceil8(C) + 3*ceil8(C)) bytes, so C <= 46), a parallel C whose image and banks exceed it
 * (C <= 1923).  KGE_EWORKSPACE: a short workspace; nothing is written. */
typedef struct kge_acre {
  int32_t in_channels, way, first_atrous, second_atrous, third_atrous, hidden_size;
  int64_t num_rel;
  float bn0_eps, bn1_eps, bn2_eps;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* bn0_mean; const float* bn0_var;
  const float* conv1_weight; const float* conv1_bias;
  const float* conv2_weight; const float* conv2_bias;
  const float* conv3_weight; const float* conv3_bias;
  const float* W_gate_e_weight; const float* W_gate_e_bias;
  const float* bn1_weight; const float* bn1_bias; const float* bn1_mean; const float* bn1_var;
  const float* fc_weight; const float* fc_bias;
  const float* bn2_weight; const float* bn2_bias; const float* bn2_mean; const float* bn2_var;
} kge_acre_t;
int64_t kge_acre_trunk_workspace_bytes(const kge_acre_t* p, int64_t Q);
int kge_acre_trunk_fwd(const kge_acre_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                       void* workspace, int64_t workspace_bytes, void* stream);

/* ---- AcrE trunk, training mode ---------------------------------------------------------------
 * AcrE.forward up to the x.E^T product (pykg2vec/models/projection.py:706-734) with self.training == True, forward
 * and backward; replaces the reference's torch layers bn0 -> inp_drop -> three dilated convs (+ residual, or the
 * W_gate_e mix) -> bn1 -> relu -> feature_map_drop -> fc -> hidden_drop -> bn2 -> relu and their autograd.  The
 * configuration and per-query function are kge_acre_trunk_fwd's, with v = bn0(img) * noise0[q, :] in place of bn0(img):
 *   serial (way 0):   y = conv3(conv2(conv1(v))) + v;   parallel (way 1): y[c] = W_gate_e([v ; conv1..3(v)[c]])
 *   x[q,:] = relu(bn2(fc(flatten(relu(bn1(y)) * noise1[q, c])) * noise2[q, :]))
 * The Q = G * B rows are G groups of B rows (G = 2: the tail and head forwards of train_step_projection as one call);
 * every BatchNorm uses the batch statistics of its own group (bn0 one channel over B*400 values, bn1 per channel over
 * B*400, bn2 per feature over B), and the running statistics are updated group after group as G sequential
 * nn.BatchNorm calls do (momentum from the struct, unbiased variance); num_batches_tracked is the caller's.
 * Running-statistic pointers: all six set, or all NULL (no update).  rel is indexed with r as given.
 * Dropout is explicit noise, bernoulli(1 - p) / (1 - p) as torch draws it (each may be NULL = no dropout):
 *   noise0 [Q, 400] (inp_drop), noise1 [Q, C] (feature_map_drop, Dropout2d: one value per channel), noise2 [Q, 200].
 * Pointers: the shapes of kge_acre_t: ent [N,200], rel [num_rel,200], conv*_bias all three set for acre_bias or all NULL,
 * W_gate_e_* set in the parallel way and ignored in the serial one; the running statistics are the
 * six writable pointers at the end.
 * KGE_EINVAL: way not 0 / 1, an atrous rate < 1, in_channels < 1, num_rel < 1, one or two NULL conv biases, a NULL
 * required pointer, B < 2 (a one-row BatchNorm1d raises in the reference), Q not a multiple of B, or Q (parallel:
 * Q*C) beyond one call's grid.  KGE_ENOTSUP: hidden_size != 200; a serial C whose backward's shared memory exceeds
 * 227 KB, 4*(400 + 802*C + 9*C*ceil8(C) + ceil8(C)) bytes, so C <= 46 (the inference trunk's bound); a parallel
 * C > 1024.  Any atrous rate >= 1 runs, including rates beyond the 20 x 20 image.
 *
 * kge_acre_train_fwd: x [Q, 200].  Every statistic is reduced in a fixed order that does not depend on the grid, so
 * x and the running statistics are bit-reproducible.  The workspace (kge_acre_train_workspace_bytes(p, Q, B) bytes)
 * keeps what the backward reads: pass the same workspace, unmodified, to kge_acre_train_bwd, once (the backward
 * overwrites the forward's features and gate rows with their gradients).  In floats it holds
 *   Q*(400*(2 + 2C) + 200*(ceil(400C/512) + 2) + 9*C*(Cin2 + Cin3 + 1) + 5C + 2) + G*(4*C + 404)
 * rounded up per region to 64 floats, plus Q*800C for the serial way's conv1 / conv2 outputs or Q*1600C for the
 * parallel way's gate rows (Cin2 = Cin3 = C serial, 1 parallel): 78 MB at (serial, 32) and 25 MB at (parallel, 9)
 * with Q = 256, B = 128.  The statistics span the group, so the call cannot be split over Q.
 * kge_acre_train_bwd: from gx = d loss / d x [Q, 200] and the forward's x, ACCUMULATES into KGE_ACRE_TRAIN_GRADS
 * dense buffers shaped like the parameters (caller zeroes), in this order: ent, rel, bn0.weight, bn0.bias,
 * conv1.weight, conv1.bias, conv2.weight, conv2.bias, conv3.weight, conv3.bias, W_gate_e.weight, W_gate_e.bias,
 * bn1.weight, bn1.bias, fc.weight, fc.bias, bn2.weight, bn2.bias.  The slots of absent parameters (the conv biases
 * without acre_bias, W_gate_e in the serial way) must be NULL and every other slot set, else KGE_EINVAL.  The entity /
 * relation rows are scattered with float atomics (ids repeat); every other sum runs in a fixed order.  No entry
 * point allocates. */
#define KGE_ACRE_TRAIN_GRADS 18
typedef struct kge_acre_train {
  int32_t in_channels, way, first_atrous, second_atrous, third_atrous, hidden_size;
  int64_t num_rel;
  float bn0_eps, bn1_eps, bn2_eps;
  float bn0_momentum, bn1_momentum, bn2_momentum;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias;
  const float* conv1_weight; const float* conv1_bias;
  const float* conv2_weight; const float* conv2_bias;
  const float* conv3_weight; const float* conv3_bias;
  const float* W_gate_e_weight; const float* W_gate_e_bias;
  const float* bn1_weight; const float* bn1_bias;
  const float* fc_weight; const float* fc_bias;
  const float* bn2_weight; const float* bn2_bias;
  float* bn0_mean; float* bn0_var; float* bn1_mean; float* bn1_var; float* bn2_mean; float* bn2_var;
} kge_acre_train_t;
int64_t kge_acre_train_workspace_bytes(const kge_acre_train_t* p, int64_t Q, int64_t B);
int kge_acre_train_fwd(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                       const float* noise0, const float* noise1, const float* noise2, float* x, void* workspace,
                       int64_t workspace_bytes, void* stream);
int kge_acre_train_bwd(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                       const float* noise0, const float* noise1, const float* noise2, const float* gx, const float* x,
                       float* const* grads, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- ProjE_pointwise (pykg2vec/models/projection.py:128-257) ------------------------------------
 * Tables with the reference's state_dict shapes (device fp32): ent [num_ent, k], rel [num_rel, k],
 * bc1 / De1 / Dr1 / bc2 / De2 / Dr2 [1, k].  k = hidden_size <= 1024 (KGE_ENOTSUP above).
 *
 * kge_proje_trunk_fwd: f1 (direction 0, :212-219) or f2 (direction 1, :221-228; plain r, no reciprocal
 * relation) for Q queries, x[q, :] = tanh(ent[e[q]] * De + rel[r[q]] * Dr + bc), times noise[q, :] when noise
 * ([Q, k]) is not NULL.  Canonical arithmetic: fmul, fmul, fadd, fadd (no contraction), then the canonical tanh
 * (DESIGN.md §3).  Evaluation ranks x with kge_proj_rank and bias NULL (g(), :248-257).  Q = 0 is a no-op.
 *
 * kge_proje_train_step: forward(e, r, er_e2, direction) of both directions (:194-210) — the dropout noise is
 * the caller's (torch.dropout(train=True) = x * noise, noise = bernoulli(1 - p) / (1 - p); NULL: no dropout) —
 * their summed loss Criterion.multi_class (criterion.py:52-55) into loss_out[0], and the backward.  hr_t /
 * tr_h: the dense [B, num_ent] label rows the Generator yields (1 positive, -1 negative, 0 ignored); either may
 * be NULL to run one direction only (its ids may then be NULL too).  Only the nonzero labels are evaluated:
 * the reference's loss gives every zero-label entry exactly zero loss and gradient.  grads[8]: dense
 * gradient buffers in parameter_list order (ent, rel, bc1, De1, Dr1, bc2, De2, Dr2), ACCUMULATED (caller
 * zeroes; each may be NULL).  The regulariser is not included: kge_reg_l1_dense.  B = 0 writes a zero loss. */
typedef struct kge_proje {
  int32_t hidden_size;
  int64_t num_ent, num_rel;
  const float* ent; const float* rel;
  const float* bc1; const float* De1; const float* Dr1;
  const float* bc2; const float* De2; const float* Dr2;
} kge_proje_t;
int kge_proje_trunk_fwd(const kge_proje_t* p, int32_t direction, const int64_t* e, const int64_t* r, int64_t Q,
                        const float* noise, float* x, void* stream);
int kge_proje_train_step(const kge_proje_t* p, const int64_t* h, const int64_t* r, const int64_t* t, int64_t B,
                         const float* hr_t, const float* tr_h, const float* noise_tail, const float* noise_head,
                         float* const* grads, float* loss_out, void* stream);

/* ProjE_pointwise.get_reg (projection.py:189-192): an L1 sum over WHOLE tensors, not over batch rows.
 *   reg_out[0] = lmbda * sum_i sum_j |w[i][j]|   for the `count` (<= 16) tensors w[i] of n[i] floats;
 *   grad[i][j] += lmbda * sign(w[i][j])          (abs's backward: sign(0) = 0); grad or grad[i] may be NULL.
 * The sum is an fp32 reduction in no fixed order. */
int kge_reg_l1_dense(const float* const* w, float* const* grad, const int64_t* n, int32_t count, float lmbda,
                     float* reg_out, void* stream);

/* ---- TuckER (pykg2vec/models/projection.py:258-345) ---------------------------------------------
 * Tables with the reference's state_dict shapes (device fp32): ent [num_ent, d1], rel [num_rel, d2],
 * W [d2, d1*d1].  d1, d2 <= 256 (KGE_ENOTSUP above; any width below, multiples of 4 or not).  The kernels
 * replace the trunk of forward() (:310-334): the reference builds one d1 x d1 matrix PER SAMPLE
 * (rel[r] @ W.view(d2, -1), :321-323) and drops it out; here one core matrix per DISTINCT relation is built and
 * the dropout mask is applied (explicit mode) or regenerated (counter mode) inside the contraction, so no
 * [Q, d1, d1] tensor exists.  Summation orders and the mask's counter layout: DESIGN.md §3 (TuckER).
 *
 * kge_tucker_cores: M[u, :] = sum_k rel[ids[u], k] * W[k, :] for u < U, out [U, d1*d1] (:321-323 per relation):
 * one fma chain over k ascending from 0, so M[u] is bit-reproducible and independent of U and of the tiling.
 *
 * kge_tucker_trunk_fwd: for q < Q, ehat = normalize(ent[e[q]]) (* noise0[q]) (:318-320); x_pre[j] = sum_i
 * ehat[i] m1[q][i][j] M[slot[q]][i][j] (:324-326), one fma chain over i ascending; x[q] = normalize(x_pre)
 * (* noise2[q]) (:327-328).  slot[q] < U is the row of M holding the core matrix of query q's relation (not
 * checked).  noise0 / noise2: [Q, d1] or NULL.  mask NULL or mode 0: no dropout1.  mode 1: m1 = noise1 [Q, d1, d1]
 * (bernoulli(1 - p) / (1 - p)).  mode 2: element (q, i, j) is kept iff a Philox-4x32-10 draw keyed on seed at
 * counter offset + (q*d1 + i)*d1 + j is >= p, kept values are 1 / (1 - p); p = 0 is no mask.  xpre [Q, d1] and
 * nrm [Q] (both or neither): x_pre and its L2 norm, which the backward reads.
 *
 * kge_tucker_trunk_bwd: from gx = d loss / d x [Q, d1] (kge_proj_tail_bwd's grad_x) through noise2 and the
 * normalisation, grad_ent[e[q]] += the gradient through noise0 and the first normalisation, and
 * dM[slot[q]][i][j] += ehat[i] m1 g[j].  grad_ent [num_ent, d1] and dM [U, d1*d1] are ACCUMULATED with float
 * atomics (caller zeroes; each may be NULL).  The mask arguments of the forward regenerate the same mask.
 *
 * kge_tucker_cores_bwd: grad_W[k, :] += sum_u rel[ids[u], k] dM[u, :];  grad_rel[ids[u], k] += sum_ij dM[u][ij]
 * W[k][ij].  Dense buffers shaped like the parameters, accumulated (caller zeroes; each may be NULL).
 *
 * kge_tucker_mask1: the mode-2 mask values of (seed, offset, p) as [Q, d1, d1] floats (tests).
 *
 * workspace: kge_tucker_workspace_bytes(p, U) bytes for kge_tucker_cores / kge_tucker_cores_bwd (KGE_EWORKSPACE
 * when short; nothing is written).  Q = 0 / U = 0 are no-ops.  No entry point allocates. */
typedef struct kge_tucker {
  int32_t d1, d2;
  int64_t num_ent, num_rel;
  const float* ent; const float* rel; const float* W;
} kge_tucker_t;
typedef struct kge_tucker_mask {
  int32_t mode;          /* 0 none, 1 explicit (noise1), 2 counter (seed, offset, p) */
  const float* noise1;
  uint64_t seed, offset;
  float p;
} kge_tucker_mask_t;
int64_t kge_tucker_workspace_bytes(const kge_tucker_t* p, int64_t U);
int kge_tucker_cores(const kge_tucker_t* p, const int64_t* ids, int64_t U, float* M, void* workspace,
                     int64_t workspace_bytes, void* stream);
int kge_tucker_trunk_fwd(const kge_tucker_t* p, const float* M, const int64_t* e, const int64_t* slot, int64_t Q,
                         const float* noise0, const kge_tucker_mask_t* mask, const float* noise2, float* x,
                         float* xpre, float* nrm, void* stream);
int kge_tucker_trunk_bwd(const kge_tucker_t* p, const float* M, const int64_t* e, const int64_t* slot, int64_t Q,
                         const float* noise0, const kge_tucker_mask_t* mask, const float* noise2, const float* gx,
                         const float* xpre, const float* nrm, float* grad_ent, float* dM, void* stream);
int kge_tucker_cores_bwd(const kge_tucker_t* p, const int64_t* ids, int64_t U, const float* dM, float* grad_rel,
                         float* grad_W, void* workspace, int64_t workspace_bytes, void* stream);
int kge_tucker_mask1(uint64_t seed, uint64_t offset, float p, int64_t Q, int32_t d1, float* out, void* stream);

/* ---- negative sampling on the device: replaces the CPU sampler processes ----
 * process_function_pairwise / process_function_pointwise (pykg2vec/data/generator.py:42-158).
 * The positives (all training triples, generator.py:52,109) are packed as 64-bit keys
 * (h<<42 | r<<22 | t; < 2^22 entities, < 2^20 relations) into an open-addressing hash set in
 * device memory: slots[capacity], capacity = kge_tripleset_capacity(n) (power of two >= 2n).
 * kge_sample_negatives draws, for positive i and j < neg_rate, u ~ U[0,1): the TAIL is corrupted
 * when u > p (generator.py:73) else the head, p = corrupt_head_prob[r] ("bern",
 * kgcontroller.py:466-492) or 0.5 when NULL ("uniform"); the replacement entity is redrawn
 * (at most 64 times) while the corrupted triple is in the set (generator.py:76-77,86-87).
 * layout 0 (pairwise): out_* are [B*neg_rate], negatives of positive i contiguous;
 * layout 1 (pointwise): out_* are [B*(1+neg_rate)], each positive followed by its negatives,
 * out_y = +1 / -1 (generator.py:125-156).  The draw is a pure function of (seed, step, index):
 * counter-based splitmix64, reproduced bit-for-bit by the CPU oracle. */
int64_t kge_tripleset_capacity(int64_t n);
int kge_tripleset_build(const int64_t* h, const int64_t* r, const int64_t* t, int64_t n,
                        uint64_t* slots, int64_t capacity, int64_t num_ent, int64_t num_rel,
                        void* stream);
int kge_sample_negatives(const uint64_t* slots, int64_t capacity, const int64_t* pos_h,
                         const int64_t* pos_r, const int64_t* pos_t, int64_t B, int32_t neg_rate,
                         const float* corrupt_head_prob, int64_t num_ent, uint64_t seed, uint64_t step,
                         int32_t layout, int64_t* out_h, int64_t* out_r, int64_t* out_t,
                         int64_t* out_y, void* stream);

/* Number of kernels this library has launched since load (all streams); used
 * by bench.py for its gpu_launches claim. */
int64_t kge_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* KGE_B200_H */
