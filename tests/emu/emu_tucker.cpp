// tests/emu/emu_tucker.cpp — TEST INFRASTRUCTURE.  Runs TuckER's kernels of pykg2vec_b200/csrc/kge_tucker.cuh (row
// gather / scatter, the relation-level GEMMs on proj_gemm_kernel, trunk forward and backward, the mask writer) on
// the host, CUDA thread by CUDA thread (tests/emu/cuda_runtime.h), with the launch geometry of the C-ABI launchers
// in kge_proj.cu (tests/test_emu_tucker.py).  Built with -DTUCKER_RACE_MAIN it is the ThreadSanitizer race check of
// the two trunk kernels.  Not a product path: nothing in pykg2vec_b200/ can reach it.
#include <cstdio>
#include <random>

#include "kge_tucker.cuh"

namespace cuda_emu {
thread_local dim3 t_threadIdx, t_blockIdx;
dim3 g_blockDim, g_gridDim;
BlockCtx* g_block = nullptr;
std::mutex g_atomic_mu;
}  // namespace cuda_emu

namespace kge {  // host-side symbols kge_common.cuh declares (defined in kge_abi.cu in the product)
void set_error(const char*, ...) {}
int cuda_fail(cudaError_t, const char*) { return KGE_ECUDA; }
void count_launch(int) {}
int sm_count() { return 132; }
}  // namespace kge

using namespace kge;

template <int EPI>
static void run_gemm(const ProjLaunch& L) {
  cuda_emu::launch(dim3(L.gx, L.gy, L.gz), dim3(PTHREADS), [&] { proj_gemm_kernel<EPI, 4, 4>(L.g); });
}

static TuckerMask make_mask(const kge_tucker_mask_t* m) {
  TuckerMask o{};
  if (!m || m->mode == TUCKER_MASK_NONE) return o;
  if (m->mode == TUCKER_MASK_EXPLICIT) { o.mode = TUCKER_MASK_EXPLICIT; o.noise1 = m->noise1; return o; }
  if (m->p == 0.f) return o;
  o.mode = TUCKER_MASK_COUNTER; o.seed = m->seed; o.offset = m->offset;
  tucker_mask_params(m->p, &o.thresh, &o.scale);
  return o;
}

extern "C" {

// ws: tucker_workspace_floats(U, d2) floats
void emu_tucker_cores(const kge_tucker_t* p, const int64_t* ids, int64_t U, float* M, float* ws) {
  cuda_emu::launch(dim3(proj_tiles(U * p->d2, 256)), dim3(256),
                   [&] { tucker_gather_rows_kernel(p->rel, ids, U, p->d2, ws); });
  run_gemm<EPI_STORE>(tucker_plan_cores(ws, p->W, U, p->d1, p->d2, M));
}

void emu_tucker_trunk_fwd(const kge_tucker_t* p, const float* M, const int64_t* e, const int64_t* slot, int64_t Q,
                          const float* noise0, const kge_tucker_mask_t* mask, const float* noise2, float* x,
                          float* xpre, float* nrm) {
  TuckerTrunk a{};
  a.ent = p->ent; a.M = M; a.e = e; a.slot = slot; a.d1 = p->d1; a.noise0 = noise0; a.noise2 = noise2;
  a.mask = make_mask(mask); a.x = x; a.xpre = xpre; a.nrm = nrm;
  cuda_emu::launch(dim3((unsigned)Q), dim3(TUCKER_THREADS), [&] { tucker_trunk_fwd_kernel(a); });
}

void emu_tucker_trunk_bwd(const kge_tucker_t* p, const float* M, const int64_t* e, const int64_t* slot, int64_t Q,
                          const float* noise0, const kge_tucker_mask_t* mask, const float* noise2, const float* gx,
                          float* xpre, float* nrm, float* gent, float* dM) {
  TuckerTrunk a{};
  a.ent = p->ent; a.M = M; a.e = e; a.slot = slot; a.d1 = p->d1; a.noise0 = noise0; a.noise2 = noise2;
  a.mask = make_mask(mask); a.gx = gx; a.xpre = xpre; a.nrm = nrm; a.gent = gent; a.dM = dM;
  cuda_emu::launch(dim3((unsigned)Q), dim3(TUCKER_THREADS), [&] { tucker_trunk_bwd_kernel(a); });
}

void emu_tucker_cores_bwd(const kge_tucker_t* p, const int64_t* ids, int64_t U, const float* dM, float* grel,
                          float* gW, float* ws) {
  const int d1 = p->d1, d2 = p->d2;
  float* drelU = ws + U * d2;
  cuda_emu::launch(dim3(proj_tiles(U * d2, 256)), dim3(256), [&] { tucker_gather_rows_kernel(p->rel, ids, U, d2, ws); });
  run_gemm<EPI_ATOMIC>(tucker_plan_grad_W(ws, dM, U, d1, d2, gW));
  for (int64_t i = 0; i < U * d2; ++i) drelU[i] = 0.f;
  run_gemm<EPI_ATOMIC>(tucker_plan_grad_rel(dM, p->W, U, d1, d2, drelU, 8));
  cuda_emu::launch(dim3(proj_tiles(U * d2, 256)), dim3(256),
                   [&] { tucker_scatter_rows_kernel(drelU, ids, U, d2, grel); });
}

void emu_tucker_mask1(uint64_t seed, uint64_t offset, float p, int64_t Q, int d1, float* out) {
  TuckerMask m{};
  m.mode = TUCKER_MASK_COUNTER; m.seed = seed; m.offset = offset;
  tucker_mask_params(p, &m.thresh, &m.scale);
  if (p == 0.f) { m.thresh = 0u; m.scale = 1.0f; }
  const long long n = Q * (long long)d1 * d1;
  cuda_emu::launch(dim3(proj_tiles(n, 256)), dim3(256), [&] { tucker_mask1_kernel(m, n, out); });
}

}  // extern "C"

#ifdef TUCKER_RACE_MAIN
// ThreadSanitizer build: the forward (row and reductions through shared memory) and the backward (shared rows
// reused across phases, float atomics into dM and the entity gradient from queries sharing a relation and an entity)
int main(int argc, char**) {
  if (argc > 1) return 64;   // "probe": only the sanitizer runtime starts
  const int d1 = 13, d2 = 5, N = 6, R = 3, Q = 3, U = 2;
  std::mt19937 gen(7);
  std::normal_distribution<float> nd(0.f, 0.5f);
  auto rnd = [&](size_t n) { std::vector<float> v(n); for (auto& x : v) x = nd(gen); return v; };
  auto ent = rnd(N * d1), rel = rnd(R * d2), W = rnd(d2 * d1 * d1), gx = rnd(Q * d1), n0 = rnd(Q * d1), n2 = rnd(Q * d1);
  kge_tucker_t p{d1, d2, N, R, ent.data(), rel.data(), W.data()};
  std::vector<int64_t> ids = {2, 0}, e = {4, 1, 4}, slot = {1, 0, 1};
  std::vector<float> M(U * d1 * d1), ws(2 * U * d2), x(Q * d1), xpre(Q * d1), nrm(Q), gent(N * d1, 0.f),
      dM(U * d1 * d1, 0.f), grel(R * d2, 0.f), gW(d2 * d1 * d1, 0.f);
  kge_tucker_mask_t mask{TUCKER_MASK_COUNTER, nullptr, 11u, 5u, 0.3f};
  emu_tucker_cores(&p, ids.data(), U, M.data(), ws.data());
  emu_tucker_trunk_fwd(&p, M.data(), e.data(), slot.data(), Q, n0.data(), &mask, n2.data(), x.data(), xpre.data(),
                       nrm.data());
  emu_tucker_trunk_bwd(&p, M.data(), e.data(), slot.data(), Q, n0.data(), &mask, n2.data(), gx.data(), xpre.data(),
                       nrm.data(), gent.data(), dM.data());
  emu_tucker_cores_bwd(&p, ids.data(), U, dM.data(), grel.data(), gW.data(), ws.data());
  printf("%g %g\n", x[0], gW[0]);
  return 0;
}
#endif
