// tests/emu/emu_models.cpp — TEST INFRASTRUCTURE.  Host emulation (tests/emu/cuda_runtime.h: one host
// thread per CUDA thread) of the device math that lives in the product's kernel headers:
//   * score_group<MODEL, VEC, GROUPING> of kge_models.cuh with score_fwd_kernel's thread mapping
//     (8-lane group per triple, 32 triples per 256-thread CTA, idle groups shadow the last triple);
//   * grad_group<MODEL, VEC> of kge_grads.cuh with score_bwd_kernel's mapping (atomics included);
//   * project_rows_kernel / normalize_rows_kernel of kge_project.cuh.
// tests/test_emu_score.py and tests/test_emu_project.py compare with the oracle (bit for bit) and with
// the gradients the reference's own autograd produced.  Not a product path.
#include "kge_grads.cuh"
#include "kge_project.cuh"

namespace cuda_emu {
thread_local dim3 t_threadIdx, t_blockIdx;
dim3 g_blockDim, g_gridDim;
BlockCtx* g_block = nullptr;
std::mutex g_atomic_mu;
}  // namespace cuda_emu

namespace kge {
void set_error(const char*, ...) {}
int cuda_fail(cudaError_t, const char*) { return KGE_ECUDA; }
void count_launch(int) {}
int sm_count() { return 132; }
int num_tables(int) { return 0; }
}  // namespace kge

using namespace kge;

// ---- forward ----
constexpr int kMaxScratch = 4096;   // floats of per-group scratch the emulated CTA provides

template <int MODEL, int VEC>
static void score_body(ModelParams P, int grouping, const int64_t* h, const int64_t* r, const int64_t* t,
                       int64_t n, float* out, int scratch_floats) {
  __shared__ __align__(16) float smem[32 * kMaxScratch];
  float* scratch = smem + (size_t)(threadIdx.x >> 3) * scratch_floats;
  const int lane = threadIdx.x & 7;
  const int64_t g = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3);
  const bool valid = g < n;
  const int64_t gi = valid ? g : n - 1;
  TripleRows R;
  resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, h[gi], r[gi], t[gi]);
  float s;
  if (grouping == KGE_GROUP_TAIL) s = score_group<MODEL, VEC, KGE_GROUP_TAIL>(R, P, lane, scratch);
  else s = score_group<MODEL, VEC, KGE_GROUP_HEAD>(R, P, lane, scratch);
  if (valid && lane == 0) out[g] = s;
}

extern "C" int emu_score_fwd(const kge_model_t* m, int grouping, int vec, const int64_t* h, const int64_t* r,
                             const int64_t* t, int64_t n, float* out) {
  const ModelParams P = make_params(m, nullptr);
  const int sf = (int)group_scratch_floats(m);
  if (sf > kMaxScratch) return KGE_ENOTSUP;
  const dim3 grid((unsigned)((n + 31) / 32)), block(256);
#define CALL(M, V) cuda_emu::launch(grid, block, [&] { score_body<M, V>(P, grouping, h, r, t, n, out, sf); })
  KGE_DISPATCH_MODEL_VEC(m->model, vec, CALL);
#undef CALL
  return KGE_OK;
}

// ---- backward ----
constexpr int kMaxScratchBwd = 8192;


struct GradTables { float* t[KGE_MAX_TABLES]; };

template <int MODEL, int VEC>
static void bwd_body(ModelParams P, GradTables GT, const int64_t* h, const int64_t* r, const int64_t* t,
                     int64_t n, const float* gout, int scratch_floats) {
  __shared__ __align__(16) float smem[32 * kMaxScratchBwd];
  float* scratch = smem + (size_t)(threadIdx.x >> 3) * scratch_floats;
  const int lane = threadIdx.x & 7;
  const int64_t g = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3);
  const bool valid = g < n;
  const int64_t gi = valid ? g : n - 1;
  const int64_t hi = h[gi], ri = r[gi], ti = t[gi];
  TripleRows R;
  resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, hi, ri, ti);
  GradRows G;
  resolve_grad_rows<MODEL>(G, P, GT.t, hi, ri, ti);
  if (!valid) {
    for (int c = 0; c < 8; ++c) G.h[c] = G.t[c] = G.r[c] = nullptr;
  }
  if (!valid && (MODEL == KGE_SLM || MODEL == KGE_NTN || MODEL == KGE_SME || MODEL == KGE_SME_BL || MODEL == KGE_CONVKB)) return;
  grad_group<MODEL, VEC>(R, G, P, lane, gout[gi], scratch);
}

extern "C" int emu_score_bwd(const kge_model_t* m, int vec, int ntab, const int64_t* h, const int64_t* r,
                             const int64_t* t, int64_t n, const float* gout, float* const* grad_tables) {
  const ModelParams P = make_params(m, nullptr);
  GradTables GT;
  for (int k = 0; k < KGE_MAX_TABLES; ++k) GT.t[k] = (k < ntab) ? grad_tables[k] : nullptr;
  if (m->model == KGE_TRANSM) GT.t[2] = nullptr;
  const int sf = (int)group_scratch_floats_bwd(m);
  if (sf > kMaxScratchBwd) return KGE_ENOTSUP;
  const dim3 grid((unsigned)((n + 31) / 32)), block(256);
#define CALL(M, V) cuda_emu::launch(grid, block, [&] { bwd_body<M, V>(P, GT, h, r, t, n, gout, sf); })
  KGE_DISPATCH_MODEL_VEC(m->model, vec, CALL);
#undef CALL
  return KGE_OK;
}

// ---- per-relation projection ----
template <int MODEL>
static void run(const ModelParams& P, int vec, int64_t r, int64_t n, float* out) {
  const dim3 grid((unsigned)((n + 31) / 32)), block(256);
  if (vec == 4) cuda_emu::launch(grid, block, [&] { project_rows_kernel<MODEL, 4>(P, r, n, out); });
  else if (vec == 2) cuda_emu::launch(grid, block, [&] { project_rows_kernel<MODEL, 2>(P, r, n, out); });
  else cuda_emu::launch(grid, block, [&] { project_rows_kernel<MODEL, 1>(P, r, n, out); });
}

extern "C" int emu_project_entities(const kge_model_t* m, int64_t r, float* out) {
  const ModelParams P = make_params(m, nullptr);
  if (m->model == KGE_TRANSR) {
    run<KGE_TRANSR>(P, pick_vec(m, 3, m->dim, m->rel_dim), r, m->num_ent, out);
    return 0;
  }
  const int vec = pick_vec(m, m->model == KGE_TRANSH ? 3 : 4, m->dim);
  if (m->model == KGE_TRANSH) run<KGE_TRANSH>(P, vec, r, m->num_ent, out);
  else if (m->model == KGE_TRANSD) run<KGE_TRANSD>(P, vec, r, m->num_ent, out);
  else return -1;
  return 0;
}

extern "C" int emu_normalize_rows(const float* in, int64_t n, int width, int vec, float* out) {
  const dim3 grid((unsigned)((n + 31) / 32)), block(256);
  if (vec == 4) cuda_emu::launch(grid, block, [&] { normalize_rows_kernel<4>(in, n, width, out); });
  else if (vec == 2) cuda_emu::launch(grid, block, [&] { normalize_rows_kernel<2>(in, n, width, out); });
  else cuda_emu::launch(grid, block, [&] { normalize_rows_kernel<1>(in, n, width, out); });
  return 0;
}
