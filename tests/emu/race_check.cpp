// tests/emu/race_check.cpp — TEST INFRASTRUCTURE: a data-race check of the kernels' shared-memory /
// warp-level synchronisation.  The kernels of kge_models.cuh / kge_grads.cuh (score and gradient
// functions of every model), kge_proj.cuh, kge_conve.cuh and kge_project.cuh run under the host
// emulation (tests/emu/cuda_runtime.h: one host thread per CUDA thread; __syncthreads, __syncwarp
// and the shuffles are the only happens-before edges between them) in a binary built with
// -fsanitize=thread.  A missing barrier between a shared-memory write and another thread's read —
// which lock-step execution on real hardware can hide — is reported by ThreadSanitizer and fails
// tests/test_emu_races.py.
//
//   race_check score <blob>     blob = one model + triples, written by the test from a golden case
//   race_check proj             projection tail (3 CTA tiles, count, split-K gradients, BCE, labels)
//   race_check conve            ConvE inference trunk
//   race_check project          TransH / TransD entity projection
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>

#include "kge_conve.cuh"
#ifndef RACE_CHECK_MINIMAL   // the barrier-free control build only needs the projection kernels
#include "kge_grads.cuh"
#include "kge_project.cuh"
#else
#include "kge_models.cuh"
#endif

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

#ifndef RACE_CHECK_MINIMAL
constexpr int kMaxScratch = 8192;
struct GradTables { float* t[KGE_MAX_TABLES]; };

template <int MODEL, int VEC>
static void score_body(ModelParams P, int grouping, const int64_t* h, const int64_t* r, const int64_t* t,
                       int64_t n, float* out, int sf) {
  __shared__ __align__(16) float smem[32 * kMaxScratch];
  float* scratch = smem + (size_t)(threadIdx.x >> 3) * sf;
  const int lane = threadIdx.x & 7;
  const int64_t g = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3);
  const bool valid = g < n;
  const int64_t gi = valid ? g : n - 1;
  TripleRows R;
  resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, h[gi], r[gi], t[gi]);
  const float s = grouping == KGE_GROUP_TAIL ? score_group<MODEL, VEC, KGE_GROUP_TAIL>(R, P, lane, scratch)
                                             : score_group<MODEL, VEC, KGE_GROUP_HEAD>(R, P, lane, scratch);
  if (valid && lane == 0) out[g] = s;
}

template <int MODEL, int VEC>
static void bwd_body(ModelParams P, GradTables GT, const int64_t* h, const int64_t* r, const int64_t* t,
                     int64_t n, const float* gout, int sf) {
  __shared__ __align__(16) float smem[32 * kMaxScratch];
  float* scratch = smem + (size_t)(threadIdx.x >> 3) * sf;
  const int lane = threadIdx.x & 7;
  const int64_t g = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3);
  const bool valid = g < n;
  const int64_t gi = valid ? g : n - 1;
  TripleRows R;
  resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, h[gi], r[gi], t[gi]);
  GradRows G;
  resolve_grad_rows<MODEL>(G, P, GT.t, h[gi], r[gi], t[gi]);
  if (!valid)
    for (int c = 0; c < 8; ++c) G.h[c] = G.t[c] = G.r[c] = nullptr;
  if (!valid && (MODEL == KGE_SLM || MODEL == KGE_NTN || MODEL == KGE_SME || MODEL == KGE_SME_BL || MODEL == KGE_CONVKB)) return;
  grad_group<MODEL, VEC>(R, G, P, lane, gout[gi], scratch);
}

static int run_score(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) return 2;
  kge_model_t m{};
  int32_t hdr[5];
  float fl[2];
  int64_t dims[2];
  if (fread(hdr, 4, 5, f) != 5 || fread(fl, 4, 2, f) != 2 || fread(dims, 8, 2, f) != 2) return 2;
  m.model = hdr[0]; m.dim = hdr[1]; m.rel_dim = hdr[2]; m.l1_flag = hdr[3];
  const int ntab = hdr[4];
  m.margin = fl[0]; m.phase_scale = fl[1]; m.num_ent = dims[0]; m.num_rel = dims[1];
  std::vector<std::vector<float>> tabs(ntab), grads(ntab);
  for (int k = 0; k < ntab; ++k) {
    int64_t nf;
    if (fread(&nf, 8, 1, f) != 1) return 2;
    tabs[k].resize(nf); grads[k].assign(nf, 0.f);
    if (fread(tabs[k].data(), 4, nf, f) != (size_t)nf) return 2;
    m.tables[k] = tabs[k].data();
  }
  int64_t n;
  if (fread(&n, 8, 1, f) != 1) return 2;
  std::vector<int64_t> h(n), r(n), t(n);
  std::vector<float> up(n), out(n);
  if (fread(h.data(), 8, n, f) != (size_t)n || fread(r.data(), 8, n, f) != (size_t)n ||
      fread(t.data(), 8, n, f) != (size_t)n || fread(up.data(), 4, n, f) != (size_t)n) return 2;
  fclose(f);
  const ModelParams P = make_params(&m, nullptr);
  GradTables GT{};
  for (int k = 0; k < ntab; ++k) GT.t[k] = grads[k].data();
  if (m.model == KGE_TRANSM) GT.t[2] = nullptr;
  const int sf = (int)group_scratch_floats(&m), sfb = (int)group_scratch_floats_bwd(&m);
  if (sf > kMaxScratch || sfb > kMaxScratch) return 3;
  const dim3 grid((unsigned)((n + 31) / 32)), block(256);
  const int vec = 1;   // the synchronisation structure does not depend on the load width
  for (int grouping = 0; grouping < 2; ++grouping) {
#define CALL(M, V) cuda_emu::launch(grid, block, [&] { score_body<M, V>(P, grouping, h.data(), r.data(), t.data(), n, out.data(), sf); })
    KGE_DISPATCH_MODEL_VEC(m.model, vec, CALL);
#undef CALL
  }
#define CALL(M, V) cuda_emu::launch(grid, block, [&] { bwd_body<M, V>(P, GT, h.data(), r.data(), t.data(), n, up.data(), sfb); })
  KGE_DISPATCH_MODEL_VEC(m.model, vec, CALL);
#undef CALL
  return 0;
}

#endif  // RACE_CHECK_MINIMAL

static std::vector<float> rnd(size_t n, unsigned seed, float scale = 0.5f, bool positive = false) {
  std::mt19937 g(seed);
  std::normal_distribution<float> d(0.f, scale);
  std::vector<float> v(n);
  for (auto& x : v) { x = d(g); if (positive) x = std::fabs(x) + 0.1f; }
  return v;
}

template <int EPI>
static void run_gemm(const ProjLaunch& L) {
  const dim3 grid(L.gx, L.gy, L.gz);
  switch (L.tile) {
    case PROJ_TILE_128x128: cuda_emu::launch(grid, dim3(PTHREADS), [&] { proj_gemm_kernel<EPI, 8, 8>(L.g); }); break;
    case PROJ_TILE_64x128: cuda_emu::launch(grid, dim3(PTHREADS), [&] { proj_gemm_kernel<EPI, 4, 8>(L.g); }); break;
    default: cuda_emu::launch(grid, dim3(PTHREADS), [&] { proj_gemm_kernel<EPI, 4, 4>(L.g); }); break;
  }
}

static int run_proj() {
  const long long B = 70, N = 150; const int k = 40;
  auto x = rnd(B * k, 1), ent = rnd(N * k, 2), bias = rnd(N, 3), gp = rnd(B * N, 4, 0.1f);
  std::vector<float> preds(B * N), thr(B), gx(B * k, 0.f), ge(N * k, 0.f), gb(N, 0.f), labels(B * N), g2(B * N);
  std::vector<int64_t> tgt(B), ptr(B + 1), idx;
  std::vector<int> counts(B * 4, 0);
  for (long long b = 0; b < B; ++b) { tgt[b] = (b * 7) % N; ptr[b] = (int64_t)idx.size(); for (int j = 0; j < 3; ++j) idx.push_back((b * 13 + j * 31) % N); }
  ptr[B] = (int64_t)idx.size();
  for (int tile = 0; tile < 3; ++tile) {
    run_gemm<EPI_STORE>(proj_plan_fwd(x.data(), ent.data(), bias.data(), B, N, k, preds.data(), tile));
    cuda_emu::launch(dim3(proj_tiles(B, 128)), dim3(128), [&] { proj_target_kernel(x.data(), ent.data(), bias.data(), tgt.data(), (int)B, k, thr.data()); });
    run_gemm<EPI_COUNT>(proj_plan_count(x.data(), ent.data(), bias.data(), B, N, k, thr.data(), counts.data(), 0, tile));
  }
  cuda_emu::launch(dim3((unsigned)B), dim3(128), [&] {
    proj_filter_kernel(x.data(), ent.data(), bias.data(), tgt.data(), ptr.data(), idx.data(), k, thr.data(), counts.data(), 0);
  });
  run_gemm<EPI_ATOMIC>(proj_plan_grad_x(gp.data(), preds.data(), ent.data(), B, N, k, gx.data(), 12));
  run_gemm<EPI_ATOMIC>(proj_plan_grad_ent(gp.data(), preds.data(), x.data(), B, N, k, ge.data()));
  cuda_emu::launch(dim3(proj_tiles(N, 256)), dim3(256), [&] { proj_colsum_kernel(gp.data(), preds.data(), (int)B, N, gb.data()); });
  float loss = 0.f;
  memset(labels.data(), 0, labels.size() * 4);
  cuda_emu::launch(dim3((unsigned)B), dim3(128), [&] { proj_labels_kernel(nullptr, ptr.data(), idx.data(), N, labels.data()); });
  cuda_emu::launch(dim3(proj_bce_blocks(B * N, 2)), dim3(256), [&] {
    proj_bce_kernel(preds.data(), labels.data(), B * N, 0.9f, 1.0f / N, proj_bce_grad_factor(1.f, B, N), proj_bce_inv_count(B, N), &loss, g2.data());
  });
  return 0;
}

static int run_conve() {
  const int k = 48, h1 = 8, h2 = k / h1; const long long Q = 5, N = 30, R2 = 6;
  const long long F = conve_feat_width(h2, h1);
  auto ent = rnd(N * k, 1), rel = rnd(R2 * k, 2), cw = rnd(32 * 9, 3), cb = rnd(32, 4), fw = rnd(k * F, 5, 0.05f), fb = rnd(k, 6);
  auto b0w = rnd(1, 7, 1.f, true), b0b = rnd(1, 8), b0m = rnd(1, 9), b0v = rnd(1, 10, 1.f, true);
  auto b1w = rnd(32, 11, 1.f, true), b1b = rnd(32, 12), b1m = rnd(32, 13), b1v = rnd(32, 14, 1.f, true);
  std::vector<int64_t> e = {1, 5, 29, 0, 7}, r = {0, 5, 3, 2, 1};
  std::vector<float> feat(Q * F + conve_fc_slices(F) * Q * k), x(Q * k);
  ConveFeat f{};
  f.ent = ent.data(); f.rel = rel.data(); f.e = e.data(); f.r = r.data(); f.k = k; f.h2 = h2; f.h1 = h1;
  f.bn0_w = b0w.data(); f.bn0_b = b0b.data(); f.bn0_mean = b0m.data(); f.bn0_var = b0v.data(); f.bn0_eps = 1e-5f;
  f.conv_w = cw.data(); f.conv_b = cb.data();
  f.bn1_w = b1w.data(); f.bn1_b = b1b.data(); f.bn1_mean = b1m.data(); f.bn1_var = b1v.data(); f.bn1_eps = 1e-5f;
  f.feat = feat.data();
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_THREADS), [&] { conve_feature_kernel(f); });
  float* partial = feat.data() + Q * F;
  run_gemm<EPI_STORE>(conve_plan_fc(feat.data(), fw.data(), Q, F, k, partial));
  cuda_emu::launch(dim3(proj_tiles(Q * k, 256)), dim3(256), [&] { conve_fc_combine_kernel(partial, conve_fc_slices(F), Q * k, k, fb.data(), x.data()); });
  return 0;
}

#ifndef RACE_CHECK_MINIMAL
static int run_project() {
  const int d = 24; const long long N = 50, R = 3;
  auto ent = rnd(N * d, 1), rel = rnd(R * d, 2), w = rnd(R * d, 3), em = rnd(N * d, 4), rm = rnd(R * d, 5);
  std::vector<float> out(N * d);
  kge_model_t m{};
  m.dim = m.rel_dim = d; m.num_ent = N; m.num_rel = R;
  m.model = KGE_TRANSH; m.tables[0] = ent.data(); m.tables[1] = rel.data(); m.tables[2] = w.data();
  ModelParams P = make_params(&m, nullptr);
  cuda_emu::launch(dim3((unsigned)((N + 31) / 32)), dim3(256), [&] { project_rows_kernel<KGE_TRANSH, 4>(P, 1, N, out.data()); });
  m.model = KGE_TRANSD; m.tables[2] = em.data(); m.tables[3] = rm.data();
  P = make_params(&m, nullptr);
  cuda_emu::launch(dim3((unsigned)((N + 31) / 32)), dim3(256), [&] { project_rows_kernel<KGE_TRANSD, 1>(P, 2, N, out.data()); });
  const int dr = 16;
  auto mats = rnd(R * d * dr, 6, 0.3f), relr = rnd(R * dr, 7);
  std::vector<float> outr(N * dr), rhat(R * dr);
  m.model = KGE_TRANSR; m.rel_dim = dr; m.tables[1] = relr.data(); m.tables[2] = mats.data();
  P = make_params(&m, nullptr);
  cuda_emu::launch(dim3((unsigned)((N + 31) / 32)), dim3(256), [&] { project_rows_kernel<KGE_TRANSR, 4>(P, 0, N, outr.data()); });
  cuda_emu::launch(dim3(1), dim3(256), [&] { normalize_rows_kernel<4>(relr.data(), R, dr, rhat.data()); });
  return 0;
}

#endif  // RACE_CHECK_MINIMAL

int main(int argc, char** argv) {
  const std::string cmd = argc > 1 ? argv[1] : "";
#ifndef RACE_CHECK_MINIMAL
  if (cmd == "score" && argc > 2) return run_score(argv[2]);
  if (cmd == "project") return run_project();
#endif
  if (cmd == "proj") return run_proj();
  if (cmd == "conve") return run_conve();
  fprintf(stderr, "usage: race_check score <blob> | proj | conve | project\n");
  return 64;
}
