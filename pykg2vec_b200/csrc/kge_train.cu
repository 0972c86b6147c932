// kge_train.cu — fused training step for the pairwise (margin) models and the sparse
// optimizer application:  replaces, per batch, Trainer.train_step_pairwise
// (pykg2vec/utils/trainer.py:147-157: two forward passes + Criterion.pairwise_hinge),
// loss.backward() (:298) and optimizer.step() (:299) for optim.SGD / optim.Adagrad
// over dense nn.Embedding gradients.
//
//   kernel A (train_hinge_kernel): one 8-lane group per triple, the positive's and the negative's groups of
//     a pair side by side in one warp: both scores (canonical arithmetic, == forward()), the hinge term from
//     one shuffle, and for active pairs each group scatters its triple's row gradients into a zero-filled
//     dense gradient scratch G.
//   kernel B (apply_rows_kernel): for every (table, id) the batch touched, take the
//     accumulated row gradient out of G with atomicExch(.,0) — duplicates of a row see
//     zeros — and apply the optimizer to that row.  G is zero again afterwards, and
//     rows the batch did not touch are neither read nor written, which for SGD and
//     Adagrad is exactly what the dense optimizers do to zero-gradient rows.
#include "kge_grads.cuh"

namespace kge {

constexpr int kThreads = 256;
constexpr int kGroupsPerCta = kThreads / 8;

struct GradTablesT { float* t[KGE_MAX_TABLES]; };

// A training batch is a few hundred pairs of pure latency: small CTAs (4 pairs) spread B = 512 over 128 SMs.
constexpr int kHingeThreads = 64;
constexpr int kHingeGroups = kHingeThreads / 8;

// CH > 0 (TransE / TransM, 16-byte rows, ch_select(d) = CH): the triple's three rows are read once into
// registers and both the score and the gradient are computed from them.  CH = 0: the looped (not register-cached)
// forms of the score / gradient functions — with both triples of a pair cached in one group this kernel was
// 12,760 instructions and stalled on instruction fetch.  Every form has the same arithmetic order, same bits.
constexpr int hinge_ch(int model, int vec, int ch) {
  return (model == KGE_TRANSE || model == KGE_TRANSM) && vec == 4 ? ch : 0;
}

template <int MODEL, int VEC, int CH>
__global__ void __launch_bounds__(kHingeThreads)
train_hinge_kernel(ModelParams P, GradTablesT GT, const int64_t* __restrict__ ph,
                   const int64_t* __restrict__ pr, const int64_t* __restrict__ pt,
                   const int64_t* __restrict__ nh, const int64_t* __restrict__ nr,
                   const int64_t* __restrict__ nt, int64_t n, float margin,
                   float* __restrict__ loss, int scratch_floats) {
  extern __shared__ float4 smem_f4[];
  __shared__ float red[kHingeThreads / 32];
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * scratch_floats;
  const int lane = threadIdx.x & 7;
  const bool neg = (threadIdx.x >> 3) & 1;                  // group 2k: the positive, 2k + 1: its negative
  const int64_t g = (int64_t)blockIdx.x * (kHingeGroups / 2) + (threadIdx.x >> 4);
  const bool valid = g < n;                                 // (the same for both groups of a pair)
  int64_t a = 0, b = 0, c = 0;
  TripleRows R;
  float s = 0.f;
  constexpr int K = CH > 0 ? CH : 1;
  float4 A[K], Bv[K], C[K];
  if (valid) {
    a = __ldg((neg ? nh : ph) + g); b = __ldg((neg ? nr : pr) + g); c = __ldg((neg ? nt : pt) + g);
    resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, a, b, c);
    if (CH > 0) {
      const int d = P.d, nch = (d + 3) >> 2;
      load_trans_chunks<K>([&](int q) { return ld_chunk<VEC>(R.h[0], q, d); },
                           [&](int q) { return ld_chunk<VEC>(R.r[0], q, d); },
                           [&](int q) { return ld_chunk<VEC>(R.t[0], q, d); }, nch, lane, A, Bv, C);
      s = trans_distance_regs<KGE_GROUP_TAIL, K>(A, Bv, C, P.l1);
      if (MODEL == KGE_TRANSM) s = fmul(__ldg(R.r[1]), s);   // == score_group
    } else {
      prefetch_triple_rows(R, P.d, P.dr, lane);   // the row misses of the dependent phases below overlap
      s = score_group<MODEL, VEC, KGE_GROUP_TAIL, 0>(R, P, lane, scratch);
    }
  }
  const float so = __shfl_xor_sync(0xffffffffu, s, 8);      // the other triple of the pair
  const float sp = neg ? so : s, sn = neg ? s : so;
  float v = fmaxf(fsub(fadd(sp, margin), sn), 0.f);        // Criterion.pairwise_hinge, criterion.py:26-29
  if (valid && v > 0.f) {
    GradRows G;
    resolve_grad_rows<MODEL>(G, P, GT.t, a, b, c);
    const float gs = neg ? -1.f : 1.f;
    if (CH > 0) grad_trans_regs<K, VEC>(A, Bv, C, G, P.d, (P.d + 3) >> 2, lane, P.l1,
                                        MODEL == KGE_TRANSM ? gs * __ldg(R.r[1]) : gs);   // == grad_group
    else grad_group<MODEL, VEC, 0>(R, G, P, lane, gs, scratch);
  }
  if (!valid || neg || lane != 0) v = 0.f;
  // batch loss: block tree + one atomic per CTA
#pragma unroll
  for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kHingeThreads / 32; ++w) t += red[w];
    if (t != 0.f) atomicAdd(loss, t);
  }
}

// Pointwise models (Trainer.train_step_pointwise, trainer.py:176-180, with Criterion.pointwise_logistic,
// criterion.py:32-34): the loss gradient of a triple depends on its own score only,
//   d/ds_i mean_j softplus(y_j s_j) = y_i sigmoid(y_i s_i) / n ,
// so forward, loss and backward are ONE kernel: the group scores its triple, adds softplus(y s)/n to the
// batch loss and scatters y sigmoid(y s)/n * d s / d rows into the dense gradient scratch.
__device__ __forceinline__ float tl_softplus(float x) { return x > 20.f ? x : log1pf(expf(x)); }   // F.softplus, threshold 20
__device__ __forceinline__ float tl_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

template <int MODEL, int VEC>
__global__ void __launch_bounds__(kThreads)
train_logistic_kernel(ModelParams P, GradTablesT GT, const int64_t* __restrict__ h, const int64_t* __restrict__ r,
                      const int64_t* __restrict__ t, const int64_t* __restrict__ y, int64_t n,
                      float* __restrict__ loss, int scratch_floats) {
  extern __shared__ float4 smem_f4[];
  __shared__ float red[kThreads / 32];
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * scratch_floats;
  const int lane = threadIdx.x & 7;
  const int64_t g = (int64_t)blockIdx.x * kGroupsPerCta + (threadIdx.x >> 3);
  const float inv_n = 1.f / (float)n;
  float v = 0.f;
  if (g < n) {
    const int64_t a = __ldg(h + g), b = __ldg(r + g), c = __ldg(t + g);
    const float yy = (float)__ldg(y + g);
    TripleRows R;
    resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, a, b, c);
    prefetch_triple_rows(R, P.d, P.dr, lane);
    const float s = score_group<MODEL, VEC, KGE_GROUP_TAIL, 0>(R, P, lane, scratch);
    const float x = yy * s;
    v = tl_softplus(x) * inv_n;
    const float gs = (x > 20.f ? 1.f : tl_sigmoid(x)) * yy * inv_n;
    GradRows G;
    resolve_grad_rows<MODEL>(G, P, GT.t, a, b, c);
    grad_group<MODEL, VEC, 0>(R, G, P, lane, gs, scratch);
    if (lane != 0) v = 0.f;
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) sum += red[w];
    if (sum != 0.f) atomicAdd(loss, sum);
  }
}

// RotatE (Trainer.train_step_pairwise, trainer.py:147-157, with Criterion.pariwise_logistic — the
// self-adversarial loss, criterion.py:14-23): the softmax runs over the neg_rate negatives of ONE positive, so a
// warp that owns a positive and its negatives can score them, form the weights, and scatter the row gradients
// without leaving the kernel — forward + loss + backward of the whole batch in ONE launch (was: two forward
// launches, the loss kernel, two backward launches).
//   phase 1: the warp's four 8-lane groups score negatives j = g, g+4, .. (canonical arithmetic == forward())
//            into shared memory; group 0 also scores the positive
//   phase 2: the warp's softmax statistics in EXACTLY the arithmetic of selfadv_kernel (kge_loss.cu): lane-strided
//            max / sum / weighted log-sigmoid + butterflies, so the loss bits equal the unfused path's
//   phase 3: the groups re-read their triples' rows (L1/L2 hits) and scatter d loss / d score * d score / d rows
__device__ __forceinline__ float tl_logsigmoid(float x) { return x < 0.f ? x - log1pf(expf(x)) : -log1pf(expf(-x)); }

// TEAM: the threads that share a positive — a warp (4 groups; small neg_rate: 8 positives per CTA) or the whole
// CTA (32 groups; large neg_rate: as many triples in flight as the unfused launches have).
template <int MODEL, int VEC, bool CTA_TEAM>
__global__ void __launch_bounds__(kThreads)
train_selfadv_kernel(ModelParams P, GradTablesT GT, const int64_t* __restrict__ ph, const int64_t* __restrict__ pr,
                     const int64_t* __restrict__ pt, const int64_t* __restrict__ nh, const int64_t* __restrict__ nr,
                     const int64_t* __restrict__ nt, int64_t B, int neg_rate, float alpha, float* __restrict__ loss,
                     int scratch_floats) {
  extern __shared__ float4 smem_f4[];
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * scratch_floats;
  // the team's negative scores, then d loss / d score
  float* sc = reinterpret_cast<float*>(smem_f4) + (size_t)kGroupsPerCta * scratch_floats +
              (CTA_TEAM ? (size_t)0 : (size_t)(threadIdx.x >> 5) * neg_rate);
  constexpr int kTeamGroups = CTA_TEAM ? kGroupsPerCta : 4;
  const int lane = threadIdx.x & 7, wl = threadIdx.x & 31;
  const int grp = CTA_TEAM ? (threadIdx.x >> 3) : (wl >> 3);
  const int64_t i = CTA_TEAM ? (int64_t)blockIdx.x : (int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  if (i >= B) return;                                                       // whole teams leave together
  const float inv_b = 1.f / (float)B;
  float p = 0.f;
  for (int j = grp; j < neg_rate; j += kTeamGroups) {
    const int64_t e = i * neg_rate + j;
    TripleRows R;
    resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, __ldg(nh + e), __ldg(nr + e), __ldg(nt + e));
    const float s = score_group<MODEL, VEC, KGE_GROUP_TAIL, 0>(R, P, lane, scratch);
    if (lane == 0) sc[j] = s;
  }
  if (grp == 0) {
    TripleRows R;
    resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, __ldg(ph + i), __ldg(pr + i), __ldg(pt + i));
    p = score_group<MODEL, VEC, KGE_GROUP_TAIL, 0>(R, P, lane, scratch);
  }
  if (CTA_TEAM) __syncthreads(); else __syncwarp();
  if (!CTA_TEAM || threadIdx.x < 32) {   // (group 0 — the positive's — is in the team's first warp)
    float mx = -INFINITY;
    for (int j = wl; j < neg_rate; j += 32) mx = fmaxf(mx, -sc[j] * alpha);
#pragma unroll
    for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    float den = 0.f;
    for (int j = wl; j < neg_rate; j += 32) den += expf(-sc[j] * alpha - mx);
#pragma unroll
    for (int off = 16; off; off >>= 1) den += __shfl_xor_sync(0xffffffffu, den, off);
    float row = 0.f;
    for (int j = wl; j < neg_rate; j += 32) {
      const float x = sc[j];
      const float w = expf(-x * alpha - mx) / den;
      row += w * tl_logsigmoid(x);
      sc[j] = -inv_b * w * tl_sigmoid(-x);       // (only this lane reads or writes slot j in this phase)
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) row += __shfl_xor_sync(0xffffffffu, row, off);
    p = __shfl_sync(0xffffffffu, p, 0);
    if (wl == 0) atomicAdd(loss, -inv_b * (row + tl_logsigmoid(-p)));
  }
  if (CTA_TEAM) __syncthreads(); else __syncwarp();
  for (int j = grp; j < neg_rate; j += kTeamGroups) {
    const int64_t e = i * neg_rate + j;
    const int64_t a = __ldg(nh + e), b = __ldg(nr + e), c = __ldg(nt + e);
    TripleRows R;
    GradRows G;
    resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, a, b, c);
    resolve_grad_rows<MODEL>(G, P, GT.t, a, b, c);
    grad_group<MODEL, VEC, 0>(R, G, P, lane, sc[j], scratch);
  }
  if (grp == 0) {
    const int64_t a = __ldg(ph + i), b = __ldg(pr + i), c = __ldg(pt + i);
    TripleRows R;
    GradRows G;
    resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, a, b, c);
    resolve_grad_rows<MODEL>(G, P, GT.t, a, b, c);
    grad_group<MODEL, VEC, 0>(R, G, P, lane, inv_b * tl_sigmoid(p), scratch);
  }
}

// ---- sparse optimizer application ---------------------------------------------
constexpr int kMaxTasks = 48;
struct ApplyTasks {
  int ntasks;
  float* w[kMaxTasks];      // table to update
  float* g[kMaxTasks];      // its gradient scratch
  float* state[kMaxTasks];  // Adagrad: sum of squared gradients (same shape); SGD: unused
  int width[kMaxTasks];
  const int64_t* ids[kMaxTasks];
};

// optimizer 0: SGD  (w -= lr * g)                       torch.optim.SGD, trainer.py:117-121
// optimizer 1: Adagrad (s += g*g; w -= lr * g / (sqrt(s) + eps))  torch.optim.Adagrad, trainer.py:122-126
// 128-bit atomic exchange (atom.exch.b128, sm_90+): takes a whole 16-byte chunk of the
// gradient row out of the scratch in one transaction and leaves zeros behind.
KGE_DEV float4 exch_zero_b128(float* addr) {
  unsigned long long lo, hi;
  asm volatile(
      "{\n\t.reg .b128 v, o;\n\t"
      "mov.b128 v, {%2, %3};\n\t"
      "atom.global.exch.b128 o, [%4], v;\n\t"
      "mov.b128 {%0, %1}, o;\n\t}"
      : "=l"(lo), "=l"(hi) : "l"(0ull), "l"(0ull), "l"(addr) : "memory");
  float4 r;
  r.x = __uint_as_float((unsigned)(lo & 0xffffffffull)); r.y = __uint_as_float((unsigned)(lo >> 32));
  r.z = __uint_as_float((unsigned)(hi & 0xffffffffull)); r.w = __uint_as_float((unsigned)(hi >> 32));
  return r;
}

// One element of an SGD / Adagrad step in torch's single-tensor order (param.add_(grad, alpha=-lr);
// state_sum.addcmul_(grad, grad); param.addcdiv_(grad, state_sum.sqrt().add_(eps), value=-lr)).  The sparse
// (apply_rows_kernel) and the dense (apply_dense_kernel) application both call it, so they give the same bits.
template <int OPT>
KGE_DEV float apply_elem(float wv, float gv, float* s, float lr, float eps) {
  if (OPT == 0) return ffma(-lr, gv, wv);
  const float sv = ffma(gv, gv, *s);
  *s = sv;
  return fsub(wv, fmul(lr, __fdiv_rn(gv, fadd(__fsqrt_rn(sv), eps))));
}

// One 8-lane group per (task, row); 8 rows per CTA, so that the 3,072 rows of a B = 512 TransE step spread over
// every SM.  A lane's chunks of a 16-byte-aligned row go in three round trips per 8 chunks (rows up to 256 floats
// in one pass): all atomic exchanges, then the weights (and state) of the nonzero chunks, then the stores.
constexpr int kApplyThreads = 64;
constexpr int kApplyGroups = kApplyThreads / 8;
constexpr int kApplyChunks = 8;

template <int OPT>
__global__ void __launch_bounds__(kApplyThreads)
apply_rows_kernel(ApplyTasks T, int64_t n, float lr, float eps) {
  const int task = blockIdx.y;
  const int lane = threadIdx.x & 7;
  const int64_t i = (int64_t)blockIdx.x * kApplyGroups + (threadIdx.x >> 3);
  if (i >= n) return;
  const int width = T.width[task];
  const size_t off = (size_t)__ldg(T.ids[task] + i) * (size_t)width;
  float* __restrict__ w = T.w[task] + off;
  float* __restrict__ g = T.g[task] + off;
  float* __restrict__ s = (OPT == 1) ? T.state[task] + off : nullptr;
  const bool vec = ((width & 3) == 0) && ((((uintptr_t)w | (uintptr_t)g | (uintptr_t)(OPT == 1 ? s : w)) & 15) == 0);
  if (vec) {
    const int nch = width >> 2;
    for (int c0 = lane; c0 < nch; c0 += 8 * kApplyChunks) {
      float4 gv[kApplyChunks], wv[kApplyChunks], sv[kApplyChunks];
      bool nz[kApplyChunks];
#pragma unroll
      for (int k = 0; k < kApplyChunks; ++k) {
        const int c = c0 + 8 * k;
        gv[k] = c < nch ? exch_zero_b128(g + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int k = 0; k < kApplyChunks; ++k) {
        const int c = c0 + 8 * k;
        nz[k] = gv[k].x != 0.f || gv[k].y != 0.f || gv[k].z != 0.f || gv[k].w != 0.f;   // (zero beyond the row)
        if (nz[k]) {
          wv[k] = *reinterpret_cast<float4*>(w + 4 * c);
          sv[k] = (OPT == 1) ? *reinterpret_cast<float4*>(s + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int k = 0; k < kApplyChunks; ++k) {
        const int c = c0 + 8 * k;
        if (nz[k]) {
          wv[k].x = apply_elem<OPT>(wv[k].x, gv[k].x, &sv[k].x, lr, eps);
          wv[k].y = apply_elem<OPT>(wv[k].y, gv[k].y, &sv[k].y, lr, eps);
          wv[k].z = apply_elem<OPT>(wv[k].z, gv[k].z, &sv[k].z, lr, eps);
          wv[k].w = apply_elem<OPT>(wv[k].w, gv[k].w, &sv[k].w, lr, eps);
          *reinterpret_cast<float4*>(w + 4 * c) = wv[k];
          if (OPT == 1) *reinterpret_cast<float4*>(s + 4 * c) = sv[k];
        }
      }
    }
  } else {
    for (int j = lane; j < width; j += 8) {
      const float gv = atomicExch(g + j, 0.f);
      if (gv != 0.f) {
        float sv = (OPT == 1) ? s[j] : 0.f;
        w[j] = apply_elem<OPT>(w[j], gv, &sv, lr, eps);
        if (OPT == 1) s[j] = sv;
      }
    }
  }
}

int check_model(const kge_model_t* m);
int model_vec(const kge_model_t* m);

// which tables a head / relation / tail id touches, per model
static int roles(int model, int which /*0 h, 1 r, 2 t*/, int out[8]) {
  switch (model) {
    case KGE_QUATE: case KGE_OCTONIONE: {
      const int C = model == KGE_QUATE ? 4 : 8;
      for (int c = 0; c < C; ++c) out[c] = (which == 1 ? C : 0) + c;
      return C;
    }
    case KGE_ANALOGY:
      if (which == 1) { out[0] = 1; out[1] = 4; out[2] = 5; return 3; }
      out[0] = 0; out[1] = 2; out[2] = 3; return 3;
    case KGE_TRANSE: case KGE_DISTMULT: case KGE_TRANSM: case KGE_HOLE: case KGE_RESCAL:
      out[0] = which == 1 ? 1 : 0; return 1;
    case KGE_SIMPLE: case KGE_SIMPLE_IGNR:
      if (which == 1) { out[0] = 2; out[1] = 3; return 2; } out[0] = 0; out[1] = 1; return 2;
    case KGE_CP: out[0] = which; return 1;  // sub, rel, obj
    case KGE_TRANSH: if (which == 1) { out[0] = 1; out[1] = 2; return 2; } out[0] = 0; return 1;
    case KGE_TRANSR: if (which == 1) { out[0] = 1; out[1] = 2; return 2; } out[0] = 0; return 1;
    case KGE_TRANSD: if (which == 1) { out[0] = 1; out[1] = 3; return 2; } out[0] = 0; out[1] = 2; return 2;
    case KGE_ROTATE: if (which == 1) { out[0] = 2; return 1; } out[0] = 0; out[1] = 1; return 2;
    case KGE_COMPLEX: case KGE_KG2E:
      if (which == 1) { out[0] = 2; out[1] = 3; return 2; } out[0] = 0; out[1] = 1; return 2;
    default: return 0;
  }
}
static int table_width(const kge_model_t* m, int k) {
  switch (m->model) {
    case KGE_TRANSR: return k == 0 ? m->dim : (k == 1 ? m->rel_dim : m->dim * m->rel_dim);
    case KGE_RESCAL: return k == 0 ? m->dim : m->dim * m->dim;
    case KGE_ANALOGY: return k < 2 ? m->dim : m->dim / 2;
    default: return m->dim;
  }
}

int launch_apply(const kge_model_t* m, float* const* tables_rw, float* const* grad_scratch,
                 float* const* state, int optimizer, const int64_t* const* hs, const int64_t* const* rs,
                 const int64_t* const* ts, int nsets, int64_t n, float lr, float eps, cudaStream_t st) {
  ApplyTasks T;
  T.ntasks = 0;
  for (int s = 0; s < nsets; ++s) {
    const int64_t* idarr[3] = {hs[s], rs[s], ts[s]};
    for (int which = 0; which < 3; ++which) {
      int tabs[8];
      const int nt = roles(m->model, which, tabs);
      for (int q = 0; q < nt; ++q) {
        const int k = tabs[q];
        if (!grad_scratch[k] || !tables_rw[k]) continue;
        if (T.ntasks >= kMaxTasks) { set_error("too many apply tasks"); return KGE_EINVAL; }
        T.w[T.ntasks] = tables_rw[k];
        T.g[T.ntasks] = grad_scratch[k];
        T.state[T.ntasks] = state ? state[k] : nullptr;
        if (optimizer == 1 && !T.state[T.ntasks]) { set_error("Adagrad needs a state table for table %d", k); return KGE_EINVAL; }
        T.width[T.ntasks] = table_width(m, k);
        T.ids[T.ntasks] = idarr[which];
        ++T.ntasks;
      }
    }
  }
  if (T.ntasks == 0) return KGE_OK;
  const dim3 grid((unsigned)((n + kApplyGroups - 1) / kApplyGroups), (unsigned)T.ntasks);
  if (optimizer == 0) apply_rows_kernel<0><<<grid, kApplyThreads, 0, st>>>(T, n, lr, eps);
  else apply_rows_kernel<1><<<grid, kApplyThreads, 0, st>>>(T, n, lr, eps);
  KGE_CHECK_LAUNCH("apply_rows_kernel");
  return KGE_OK;
}


// Dense optimizer.step() over ONE parameter tensor (any shape, n floats): the accumulated gradient
// is taken out of `g` (left zero-filled, ready for the next step's atomics) and applied in place.
//   OPT 0 torch.optim.SGD      w -= lr * g                                   (trainer.py:117-121)
//   OPT 1 torch.optim.Adagrad  s += g*g ; w -= lr * g / (sqrt(s) + eps)      (trainer.py:122-126)
//   OPT 2 torch.optim.Adam     m += (g - m)(1 - b1) ; v = v*b2 + (1 - b2) g*g ;
//                              w -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)   (trainer.py:112-116)
// Adam moves EVERY element every step (the moments of rows without gradient keep decaying and keep
// pushing the weight), exactly as the dense reference optimizer does — which is why this is a sweep
// over the whole tensor and not a sparse row update.  HBM-bound: 16-32 bytes per element.
template <int OPT>
__global__ void __launch_bounds__(256)
apply_dense_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ s1, float* __restrict__ s2,
                   int64_t n4, int64_t n, float lr, float eps, float b1, float b2, float step_size, float bc2_sqrt) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 gv = reinterpret_cast<float4*>(g)[i];
    if (OPT != 2 && gv.x == 0.f && gv.y == 0.f && gv.z == 0.f && gv.w == 0.f) continue;   // SGD / Adagrad: nothing moves
    float4 wv = reinterpret_cast<float4*>(w)[i];
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (OPT >= 1) a = reinterpret_cast<float4*>(s1)[i];
    if (OPT == 2) b = reinterpret_cast<float4*>(s2)[i];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float gg = f4_get(gv, e);
      float& ww = f4_at(wv, e);
      if (OPT <= 1) {
        ww = apply_elem<OPT>(ww, gg, &f4_at(a, e), lr, eps);
      } else {
        float& m = f4_at(a, e);
        float& v = f4_at(b, e);
        m = ffma(fsub(gg, m), 1.0f - b1, m);                       // exp_avg.lerp_(grad, 1 - beta1)
        v = ffma(fmul(gg, gg), 1.0f - b2, fmul(v, b2));            // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
        const float denom = fadd(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
        ww = ffma(-step_size, __fdiv_rn(m, denom), ww);            // param.addcdiv_(exp_avg, denom, value = -step_size)
      }
    }
    reinterpret_cast<float4*>(w)[i] = wv;
    if (OPT >= 1) reinterpret_cast<float4*>(s1)[i] = a;
    if (OPT == 2) reinterpret_cast<float4*>(s2)[i] = b;
    reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  // scalar tail (n % 4 elements), handled by the first threads of block 0
  const int64_t tail0 = n4 * 4;
  if (blockIdx.x == 0 && threadIdx.x < (unsigned)(n - tail0)) {
    const int64_t i = tail0 + threadIdx.x;
    const float gg = g[i];
    float ww = w[i];
    if (OPT <= 1) {
      if (gg != 0.f) {   // SGD / Adagrad: nothing moves
        float ss = OPT == 1 ? s1[i] : 0.f;
        ww = apply_elem<OPT>(ww, gg, &ss, lr, eps);
        if (OPT == 1) s1[i] = ss;
      }
    } else {
      const float m = ffma(fsub(gg, s1[i]), 1.0f - b1, s1[i]);
      const float v = ffma(fmul(gg, gg), 1.0f - b2, fmul(s2[i], b2));
      s1[i] = m; s2[i] = v;
      ww = ffma(-step_size, __fdiv_rn(m, fadd(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps)), ww);
    }
    w[i] = ww;
    g[i] = 0.f;
  }
}

}  // namespace kge

using namespace kge;

extern "C" int kge_train_pairwise_hinge_sgd(const kge_model_t* m, float* const* tables_rw,
                                            float* const* grad_scratch, const int64_t* pos_h,
                                            const int64_t* pos_r, const int64_t* pos_t,
                                            const int64_t* neg_h, const int64_t* neg_r,
                                            const int64_t* neg_t, int64_t n, float margin, float lr,
                                            float* loss_out, void* stream) {
  int rc = check_model(m);
  if (rc) return rc;
  if (n <= 0 || !tables_rw || !grad_scratch || !pos_h || !pos_r || !pos_t || !neg_h || !neg_r || !neg_t || !loss_out) {
    set_error("kge_train_pairwise_hinge_sgd: bad arguments"); return KGE_EINVAL;
  }
  const int nt = num_tables(m->model);
  const ModelParams P = make_params(m, nullptr);
  GradTablesT GT;
  int vec = model_vec(m);
  for (int k = 0; k < KGE_MAX_TABLES; ++k) {
    GT.t[k] = (k < nt) ? grad_scratch[k] : nullptr;
    if (k < nt && m->model == KGE_TRANSM && k == 2) GT.t[k] = nullptr;
    if (GT.t[k]) {
      if ((const float*)tables_rw[k] != m->tables[k]) { set_error("tables_rw[%d] must alias m->tables[%d]", k, k); return KGE_EINVAL; }
      const uintptr_t a = (uintptr_t)GT.t[k];
      if (vec == 4 && (a & 15)) vec = 2;
      if (vec == 2 && (a & 7)) vec = 1;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  KGE_CUDA_OK(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  const int sf = (int)group_scratch_floats_bwd(m);
  const size_t smem = (size_t)sf * kHingeGroups * sizeof(float);
  const unsigned grid = (unsigned)((n + kHingeGroups / 2 - 1) / (kHingeGroups / 2));
  const int ch = hinge_ch(m->model, vec, ch_select(m->dim));
#define LAUNCH(M, V, C)                                                                           \
  do {                                                                                            \
    if (smem > 40 * 1024)                                                                         \
      KGE_CUDA_OK(cudaFuncSetAttribute(train_hinge_kernel<M, V, C>,                               \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));  \
    train_hinge_kernel<M, V, C><<<grid, kHingeThreads, smem, st>>>(P, GT, pos_h, pos_r, pos_t, neg_h, neg_r, \
                                                                   neg_t, n, margin, loss_out, sf); \
  } while (0)
#define CALL(M, V)                                             \
  do {                                                         \
    if (ch == 2) { LAUNCH(M, V, hinge_ch(M, V, 2)); }          \
    else if (ch == 4) { LAUNCH(M, V, hinge_ch(M, V, 4)); }     \
    else if (ch == 8) { LAUNCH(M, V, hinge_ch(M, V, 8)); }     \
    else { LAUNCH(M, V, 0); }                                  \
  } while (0)
  KGE_DISPATCH_MODEL_VEC(m->model, vec, CALL);
#undef CALL
#undef LAUNCH
  KGE_CHECK_LAUNCH("train_hinge_kernel");
  const int64_t* hs[2] = {pos_h, neg_h};
  const int64_t* rs[2] = {pos_r, neg_r};
  const int64_t* ts[2] = {pos_t, neg_t};
  float* gs[KGE_MAX_TABLES];
  for (int k = 0; k < KGE_MAX_TABLES; ++k) gs[k] = GT.t[k];
  return launch_apply(m, tables_rw, gs, nullptr, 0, hs, rs, ts, 2, n, lr, 0.f, st);
}

extern "C" int kge_optim_apply_rows(const kge_model_t* m, float* const* tables_rw,
                                    float* const* grad_scratch, float* const* state, int optimizer,
                                    const int64_t* h, const int64_t* r, const int64_t* t, int64_t n,
                                    float lr, float eps, void* stream) {
  int rc = check_model(m);
  if (rc) return rc;
  if (n <= 0 || !tables_rw || !grad_scratch || !h || !r || !t || (optimizer != 0 && optimizer != 1)) {
    set_error("kge_optim_apply_rows: bad arguments"); return KGE_EINVAL;
  }
  float* gs[KGE_MAX_TABLES];
  const int nt = num_tables(m->model);
  for (int k = 0; k < KGE_MAX_TABLES; ++k) gs[k] = (k < nt) ? grad_scratch[k] : nullptr;
  if (m->model == KGE_TRANSM) gs[2] = nullptr;
  const int64_t* hs[1] = {h};
  const int64_t* rs[1] = {r};
  const int64_t* ts[1] = {t};
  return launch_apply(m, tables_rw, gs, state, optimizer, hs, rs, ts, 1, n, lr, eps, (cudaStream_t)stream);
}

extern "C" int kge_optim_apply_dense(float* w, float* grad, float* state1, float* state2, int64_t n, int optimizer,
                                     float lr, float eps, float beta1, float beta2, int64_t step, void* stream) {
  if (!w || !grad || n < 0 || optimizer < 0 || optimizer > 2 || (optimizer >= 1 && !state1) ||
      (optimizer == 2 && (!state2 || step < 1))) {
    set_error("kge_optim_apply_dense: bad arguments"); return KGE_EINVAL;
  }
  if (n == 0) return KGE_OK;
  if (((uintptr_t)w | (uintptr_t)grad | (uintptr_t)state1 | (uintptr_t)state2) & 15) {
    set_error("kge_optim_apply_dense: tensors must be 16-byte aligned"); return KGE_EINVAL;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n4 = n / 4;
  int64_t blocks = (n4 + 255) / 256;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  // bias corrections in double, as torch computes them in Python floats
  const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
  const float step_size = optimizer == 2 ? (float)((double)lr / bc1) : 0.f;
  const float bc2_sqrt = optimizer == 2 ? (float)sqrt(bc2) : 1.f;
  if (optimizer == 0)
    apply_dense_kernel<0><<<(unsigned)blocks, 256, 0, st>>>(w, grad, state1, state2, n4, n, lr, eps, beta1, beta2, step_size, bc2_sqrt);
  else if (optimizer == 1)
    apply_dense_kernel<1><<<(unsigned)blocks, 256, 0, st>>>(w, grad, state1, state2, n4, n, lr, eps, beta1, beta2, step_size, bc2_sqrt);
  else
    apply_dense_kernel<2><<<(unsigned)blocks, 256, 0, st>>>(w, grad, state1, state2, n4, n, lr, eps, beta1, beta2, step_size, bc2_sqrt);
  KGE_CHECK_LAUNCH("apply_dense_kernel");
  return KGE_OK;
}

extern "C" int kge_train_pointwise_logistic(const kge_model_t* m, float* const* grad_scratch, const int64_t* h,
                                            const int64_t* r, const int64_t* t, const int64_t* y, int64_t n,
                                            float* loss_out, void* stream) {
  int rc = check_model(m);
  if (rc) return rc;
  if (n <= 0 || !grad_scratch || !h || !r || !t || !y || !loss_out) {
    set_error("kge_train_pointwise_logistic: bad arguments"); return KGE_EINVAL;
  }
  switch (m->model) {   // the pointwise (logistic) row models of pointwise.py
    case KGE_DISTMULT: case KGE_COMPLEX: case KGE_CP: case KGE_SIMPLE: case KGE_SIMPLE_IGNR: case KGE_ANALOGY:
    case KGE_QUATE: case KGE_OCTONIONE: break;
    default: set_error("kge_train_pointwise_logistic: model %d is not a pointwise row model", (int)m->model); return KGE_ENOTSUP;
  }
  const int nt = num_tables(m->model);
  const ModelParams P = make_params(m, nullptr);
  GradTablesT GT;
  int vec = model_vec(m);
  for (int k = 0; k < KGE_MAX_TABLES; ++k) {
    GT.t[k] = (k < nt) ? grad_scratch[k] : nullptr;
    if (GT.t[k]) {
      const uintptr_t a = (uintptr_t)GT.t[k];
      if (vec == 4 && (a & 15)) vec = 2;
      if (vec == 2 && (a & 7)) vec = 1;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  KGE_CUDA_OK(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  const int sf = (int)group_scratch_floats_bwd(m);
  const size_t smem = (size_t)sf * kGroupsPerCta * sizeof(float);
  const unsigned grid = (unsigned)((n + kGroupsPerCta - 1) / kGroupsPerCta);
#define CALL_TL(M, V)                                                                            \
  do {                                                                                           \
    if (smem > 40 * 1024)                                                                        \
      KGE_CUDA_OK(cudaFuncSetAttribute(train_logistic_kernel<M, V>,                              \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    train_logistic_kernel<M, V><<<grid, kThreads, smem, st>>>(P, GT, h, r, t, y, n, loss_out, sf); \
  } while (0)
  switch (m->model) {
    case KGE_DISTMULT: KGE_DISPATCH_VEC(KGE_DISTMULT, vec, CALL_TL); break;
    case KGE_COMPLEX: KGE_DISPATCH_VEC(KGE_COMPLEX, vec, CALL_TL); break;
    case KGE_CP: KGE_DISPATCH_VEC(KGE_CP, vec, CALL_TL); break;
    case KGE_SIMPLE: KGE_DISPATCH_VEC(KGE_SIMPLE, vec, CALL_TL); break;
    case KGE_SIMPLE_IGNR: KGE_DISPATCH_VEC(KGE_SIMPLE_IGNR, vec, CALL_TL); break;
    case KGE_ANALOGY: KGE_DISPATCH_VEC(KGE_ANALOGY, vec, CALL_TL); break;
    case KGE_QUATE: KGE_DISPATCH_VEC(KGE_QUATE, vec, CALL_TL); break;
    default: KGE_DISPATCH_VEC(KGE_OCTONIONE, vec, CALL_TL); break;
  }
#undef CALL_TL
  KGE_CHECK_LAUNCH("train_logistic_kernel");
  return KGE_OK;
}

extern "C" int kge_train_pairwise_selfadv(const kge_model_t* m, float* const* grad_scratch, const int64_t* pos_h,
                                          const int64_t* pos_r, const int64_t* pos_t, const int64_t* neg_h,
                                          const int64_t* neg_r, const int64_t* neg_t, int64_t B, int32_t neg_rate,
                                          float alpha, float* loss_out, void* stream) {
  int rc = check_model(m);
  if (rc) return rc;
  if (B <= 0 || neg_rate <= 0 || !grad_scratch || !pos_h || !pos_r || !pos_t || !neg_h || !neg_r || !neg_t || !loss_out) {
    set_error("kge_train_pairwise_selfadv: bad arguments"); return KGE_EINVAL;
  }
  if (m->model != KGE_ROTATE) {   // the reference uses this loss for RotatE only (trainer.py:152-155)
    set_error("kge_train_pairwise_selfadv: model %d does not train with the self-adversarial loss", (int)m->model);
    return KGE_ENOTSUP;
  }
  const int nt = num_tables(m->model);
  const ModelParams P = make_params(m, nullptr);
  GradTablesT GT;
  int vec = model_vec(m);
  for (int k = 0; k < KGE_MAX_TABLES; ++k) {
    GT.t[k] = (k < nt) ? grad_scratch[k] : nullptr;
    if (GT.t[k]) {
      const uintptr_t a = (uintptr_t)GT.t[k];
      if (vec == 4 && (a & 15)) vec = 2;
      if (vec == 2 && (a & 7)) vec = 1;
    }
  }
  const int sf = (int)group_scratch_floats_bwd(m);
  // a warp per positive while each of its 4 groups has at most one negative; beyond that the whole CTA shares a
  // positive (at neg_rate 16 the warp form runs 4 triples in sequence per group, twice, while the CTA form spreads
  // them over the CTA; profiles/selfadv_fusion_probe.py times both against the five-launch path)
  const bool cta_team = neg_rate > 4;
  const size_t smem = ((size_t)sf * kGroupsPerCta + (size_t)(cta_team ? 1 : kThreads / 32) * (size_t)neg_rate) * sizeof(float);
  if (smem > 200 * 1024) {
    set_error("kge_train_pairwise_selfadv: neg_rate %d needs %zu bytes of shared memory per CTA", (int)neg_rate, smem);
    return KGE_ENOTSUP;
  }
  cudaStream_t st = (cudaStream_t)stream;
  KGE_CUDA_OK(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  const unsigned grid = cta_team ? (unsigned)B : (unsigned)((B + kThreads / 32 - 1) / (kThreads / 32));
#define CALL_SA2(M, V, T)                                                                        \
  do {                                                                                           \
    if (smem > 40 * 1024)                                                                        \
      KGE_CUDA_OK(cudaFuncSetAttribute(train_selfadv_kernel<M, V, T>,                            \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    train_selfadv_kernel<M, V, T><<<grid, kThreads, smem, st>>>(P, GT, pos_h, pos_r, pos_t, neg_h, neg_r, neg_t, B, \
                                                                (int)neg_rate, alpha, loss_out, sf); \
  } while (0)
#define CALL_SA(M, V) do { if (cta_team) CALL_SA2(M, V, true); else CALL_SA2(M, V, false); } while (0)
  KGE_DISPATCH_VEC(KGE_ROTATE, vec, CALL_SA);
#undef CALL_SA
#undef CALL_SA2
  KGE_CHECK_LAUNCH("train_selfadv_kernel");
  return KGE_OK;
}
