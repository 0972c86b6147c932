// kge_proje.cuh — kernels of ProjE_pointwise (pykg2vec/models/projection.py:128-257), launched from kge_proj.cu.
//   proje_trunk_kernel     f1 / f2 (:212-228), optionally times a dropout noise: the operand x of g() (:248-257)
//   proje_step_kernel      forward + loss (:194-210) + backward of one (row, direction) per CTA, over the
//                          LABELLED entries of the row only
//   proj_labels_neg_kernel the -1 labels of process_function_multiclass with neg_rate > 0 (generator.py:211-238)
//   reg_l1_kernel          get_reg (:189-192): an L1 sum over whole tables, and lmbda * sign(w) into their gradients
//
// Why only the labelled entries: the loss (:205-208) multiplies every term by max(0, y) or max(0, -y), so an
// entity whose label is 0 adds exactly 0 to the loss and to every gradient.  A row's nonzero labels are its
// positives and the <= 100 shared negatives of the batch: ~B (|pos| + 100) dot products replace the B x N
// product against every entity and the four dense [B,N] x [N,k] GEMMs of its backward.
//
// Canonical arithmetic (DESIGN.md §3, ProjE):
//   x[j]    = tanh_canon(fadd(fadd(fmul(e[j], De[j]), fmul(r[j], Dr[j])), bc[j]))   then fmul(x[j], noise[j])
//             (the reference's separate ATen ops h*De, r*Dr, +, +bc, tanh, dropout's multiply; no contraction)
//   logit   = ONE sequential fma chain over j from 0 of x[j] * E[n][j] (rule 8: == kge_proj_tail_fwd's logit)
//   s       = sigmoid_canon(logit);  o = fsub(1, s)
//   loss   -= log(clamp(s, 1e-10, 1)) * max(0, y) + log(clamp(o, 1e-10, 1)) * max(0, -y)
//   ds      = (-max(0,y)) / clamp(s)  [where 1e-10 <= s <= 1, else 0]  +  max(0,-y) / clamp(o)  [likewise on o]
//   g       = fmul(fmul(ds, o), s)                      (torch's sigmoid backward order)
// x, logit and g are per-element and bit-exact against tests/oracle_proje; the sums over entries (d loss / d x,
// the entity-gradient scatter, the loss) are float atomics / reductions in no fixed order.
#pragma once
#include "kge_proj.cuh"

namespace kge {

constexpr int PROJE_THREADS = 256;
constexpr int PROJE_MAX_K = 1024;   // widest row a CTA keeps in shared memory
constexpr int PROJE_WIN = 1024;     // label entries scanned per pass (4 per thread, coalesced)
constexpr int PROJE_CAP = 2048;     // labelled entries held before they are processed

KGE_DEV float proje_pre(float ev, float rv, float De, float Dr, float bc) {
  return tanh_canon(fadd(fadd(fmul(ev, De), fmul(rv, Dr)), bc));
}

// x[q, :] for Q queries of one direction: De / Dr / bc are De1 / Dr1 / bc1 (tail, f1) or De2 / Dr2 / bc2 (head, f2)
__global__ void __launch_bounds__(256)
proje_trunk_kernel(const float* __restrict__ ent, const float* __restrict__ rel, const float* __restrict__ De,
                   const float* __restrict__ Dr, const float* __restrict__ bc, const int64_t* __restrict__ e,
                   const int64_t* __restrict__ r, long long Q, int k, const float* __restrict__ noise,
                   float* __restrict__ x) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= Q * k) return;
  const long long q = i / k;
  const int j = (int)(i - q * k);
  float v = proje_pre(__ldg(ent + __ldg(e + q) * k + j), __ldg(rel + __ldg(r + q) * k + j), __ldg(De + j),
                      __ldg(Dr + j), __ldg(bc + j));
  if (noise) v = fmul(v, __ldg(noise + i));
  x[i] = v;
}

struct ProjeDir {           // one direction: f1 (tail, d = 0) or f2 (head, d = 1)
  const int64_t* e;         // h (tail) or t (head), [B]
  const float* labels;      // dense [B, N] label rows (hr_t / tr_h)
  const float* noise;       // [B, k] dropout noise or NULL
  const float* De; const float* Dr; const float* bc;
  float* gDe; float* gDr; float* gbc;   // [k] gradients, accumulated (each may be NULL)
};

struct ProjeStep {
  const float* ent; const float* rel;
  const int64_t* r;
  long long N; int k, B;
  ProjeDir dir[2];
  int dirs[2];              // direction of blockIdx.y
  float* gent; float* grel; // dense [N,k] / [R,k] gradients, accumulated (each may be NULL)
  float* loss;              // += the loss (the launcher zeroes it)
  float* dbg_logit;         // tests only (tests/emu): [2][B][N] logit and g of every labelled entry; NULL here
  float* dbg_g;
};

// one CTA per (row b, direction): x in shared memory, the label row scanned in windows of PROJE_WIN entries and
// its nonzero entries compacted into a list that is processed whenever it could overflow on the next window
__global__ void __launch_bounds__(PROJE_THREADS) proje_step_kernel(const ProjeStep s) {
  __shared__ float xs[PROJE_MAX_K];   // x after dropout
  __shared__ float ts[PROJE_MAX_K];   // tanh output
  __shared__ float gx[PROJE_MAX_K];   // d loss / d x (after dropout)
  __shared__ int lid[PROJE_CAP];      // labelled entity ids of the list
  __shared__ float lv[PROJE_CAP];     // their labels, then their g
  __shared__ int cnt;
  __shared__ float red[PROJE_THREADS / 32];
  const int tid = threadIdx.x, k = s.k, b = blockIdx.x, d = s.dirs[blockIdx.y];
  const ProjeDir& P = s.dir[d];
  const long long N = s.N;
  const int64_t eid = __ldg(P.e + b), rid = __ldg(s.r + b);
  const float* er = s.ent + eid * k;
  const float* rr = s.rel + rid * k;
  const float* nz = P.noise ? P.noise + (long long)b * k : nullptr;
  for (int j = tid; j < k; j += PROJE_THREADS) {
    const float t = proje_pre(__ldg(er + j), __ldg(rr + j), __ldg(P.De + j), __ldg(P.Dr + j), __ldg(P.bc + j));
    ts[j] = t;
    xs[j] = nz ? fmul(t, __ldg(nz + j)) : t;
    gx[j] = 0.f;
  }
  if (tid == 0) cnt = 0;
  __syncthreads();
  const float* lab = P.labels + (long long)b * N;
  const bool vec = (k % 4 == 0) && (((uintptr_t)s.ent & 15) == 0);
  float loss = 0.f;
  for (long long w0 = 0; w0 < N; w0 += PROJE_WIN) {
#pragma unroll
    for (int u = 0; u < PROJE_WIN / PROJE_THREADS; ++u) {
      const long long n = w0 + u * PROJE_THREADS + tid;
      if (n < N) {
        const float y = __ldg(lab + n);
        if (y != 0.f) {
          const int p = atomicAdd(&cnt, 1);
          lid[p] = (int)n;
          lv[p] = y;
        }
      }
    }
    __syncthreads();
    const int c = cnt;
    __syncthreads();   // every thread has read cnt before it is reset or grows again
    if (c > PROJE_CAP - PROJE_WIN || w0 + PROJE_WIN >= N) {
      // (1) one thread per labelled entry: logit, sigmoid, loss terms, g
      for (int i = tid; i < c; i += PROJE_THREADS) {
        const int n = lid[i];
        const float y = lv[i];
        const float* en = s.ent + (long long)n * k;
        float acc = 0.f;
        if (vec) {
          for (int q = 0; q < k / 4; ++q) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(en) + q);
            acc = ffma(xs[4 * q + 0], v.x, acc);
            acc = ffma(xs[4 * q + 1], v.y, acc);
            acc = ffma(xs[4 * q + 2], v.z, acc);
            acc = ffma(xs[4 * q + 3], v.w, acc);
          }
        } else {
          for (int j = 0; j < k; ++j) acc = ffma(xs[j], __ldg(en + j), acc);
        }
        const float sg = sigmoid_canon(acc);
        const float om = fsub(1.0f, sg);
        const float wl = y > 0.f ? y : 0.f, wr = -y > 0.f ? -y : 0.f;
        const float c1 = fminf(fmaxf(sg, 1e-10f), 1.0f), c2 = fminf(fmaxf(om, 1e-10f), 1.0f);
        loss = fsub(loss, fadd(fmul(log_canon(c1), wl), fmul(log_canon(c2), wr)));
        const float gl = (sg >= 1e-10f && sg <= 1.0f) ? __fdiv_rn(-wl, c1) : 0.f;
        const float gr = (om >= 1e-10f && om <= 1.0f) ? __fdiv_rn(wr, c2) : 0.f;
        const float g = fmul(fmul(fadd(gl, gr), om), sg);
        lv[i] = g;
        if (s.dbg_logit) {
          const long long o = ((long long)d * s.B + b) * N + n;
          s.dbg_logit[o] = acc;
          s.dbg_g[o] = g;
        }
      }
      __syncthreads();
      // (2) one thread per feature j: d loss / d x[j] += g E[n][j], and the scatter dE[n][j] += g x[j]
      for (int j = tid; j < k; j += PROJE_THREADS) {
        const float xj = xs[j];
        float a = gx[j];
        for (int i = 0; i < c; ++i) {
          const float g = lv[i];
          if (g == 0.f) continue;
          const long long o = (long long)lid[i] * k + j;
          a = ffma(g, __ldg(s.ent + o), a);
          if (s.gent) atomicAdd(s.gent + o, fmul(g, xj));
        }
        gx[j] = a;
      }
      if (tid == 0) cnt = 0;
      __syncthreads();
    }
  }
  // back through the dropout multiply and tanh (1 - t^2) into the two gathered rows and De / Dr / bc
  for (int j = tid; j < k; j += PROJE_THREADS) {
    const float gxd = nz ? fmul(gx[j], __ldg(nz + j)) : gx[j];
    const float t = ts[j];
    const float gp = fmul(gxd, fsub(1.0f, fmul(t, t)));
    if (gp == 0.f) continue;
    if (s.gent) atomicAdd(s.gent + eid * k + j, fmul(gp, __ldg(P.De + j)));
    if (s.grel) atomicAdd(s.grel + rid * k + j, fmul(gp, __ldg(P.Dr + j)));
    if (P.gDe) atomicAdd(P.gDe + j, fmul(gp, __ldg(er + j)));
    if (P.gDr) atomicAdd(P.gDr + j, fmul(gp, __ldg(rr + j)));
    if (P.gbc) atomicAdd(P.gbc + j, gp);
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, off);
  if ((tid & 31) == 0) red[tid >> 5] = loss;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < PROJE_THREADS / 32; ++w) t += red[w];
    atomicAdd(s.loss, t);
  }
}

// labels[b, neg[j]] = -1 wherever it is still 0 (the positives keep their 1), one CTA per row
__global__ void __launch_bounds__(128)
proj_labels_neg_kernel(float* __restrict__ labels, long long N, const int64_t* __restrict__ neg, int nneg) {
  float* row = labels + (long long)blockIdx.x * N;
  for (int j = threadIdx.x; j < nneg; j += blockDim.x) {
    float* p = row + __ldg(neg + j);
    if (*p == 0.f) *p = -1.0f;
  }
}

struct L1Seg { const float* w; float* g; long long n; };
struct L1Args { L1Seg seg[KGE_MAX_TABLES]; float lmbda; float* out; };

// blockIdx.y = segment: out += lmbda * sum |w|;  g += lmbda * sign(w)   (abs backward: sgn, sign(0) = 0)
__global__ void __launch_bounds__(256) reg_l1_kernel(const L1Args a) {
  __shared__ float red[8];
  const L1Seg S = a.seg[blockIdx.y];
  const float lm = a.lmbda;
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < S.n; i += (long long)gridDim.x * 256) {
    const float w = S.w[i];
    acc = fadd(acc, fabsf(w));
    if (S.g) S.g[i] = fadd(S.g[i], w > 0.f ? lm : (w < 0.f ? -lm : 0.f));
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w];
    if (t != 0.f) atomicAdd(a.out, fmul(t, lm));
  }
}

inline unsigned reg_l1_blocks(long long nmax, int sms) {
  const long long blocks = (nmax + 255) / 256, cap = 4ll * sms;
  return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

}  // namespace kge
