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

#define KGE_ABI_VERSION 5
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
 * batch moves B ids instead of B*N floats over PCIe.  (The -1 entries the reference adds when
 * neg_rate > 0, used by ProjE only, are not produced.) */
int kge_proj_labels(const int64_t* rows, const int64_t* ptr, const int64_t* idx, int64_t B, int64_t N,
                    float* labels, void* stream);

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
 * Training (batch statistics, dropout, autograd) stays with the framework's own layers. */
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
