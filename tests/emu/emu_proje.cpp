// tests/emu/emu_proje.cpp — TEST INFRASTRUCTURE.  Runs ProjE_pointwise's kernels of
// pykg2vec_b200/csrc/kge_proje.cuh (trunk, training step, negative labels, L1 regulariser) on the host, CUDA
// thread by CUDA thread (tests/emu/cuda_runtime.h), with the launch geometry of the C-ABI launchers in
// kge_proj.cu (tests/test_emu_proje.py).  Not a product path: nothing in pykg2vec_b200/ can reach it.
#include "kge_proje.cuh"

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

extern "C" {

void emu_proje_trunk(const kge_proje_t* p, int dir, const int64_t* e, const int64_t* r, int64_t Q, const float* noise,
                     float* x) {
  const int k = p->hidden_size;
  cuda_emu::launch(dim3(proj_tiles(Q * k, 256)), dim3(256), [&] {
    proje_trunk_kernel(p->ent, p->rel, dir ? p->De2 : p->De1, dir ? p->Dr2 : p->Dr1, dir ? p->bc2 : p->bc1, e, r, Q, k,
                       noise, x);
  });
}

// kge_proje_train_step's launch; dbg_logit / dbg_g ([2][B][N], may be NULL) receive every labelled entry's
// logit and g
void emu_proje_step(const kge_proje_t* p, const int64_t* h, const int64_t* r, const int64_t* t, int64_t B,
                    const float* hr_t, const float* tr_h, const float* noise_tail, const float* noise_head,
                    float* const* grads, float* loss, float* dbg_logit, float* dbg_g) {
  ProjeStep s{};
  s.ent = p->ent; s.rel = p->rel; s.r = r; s.N = p->num_ent; s.k = p->hidden_size; s.B = (int)B;
  s.gent = grads[0]; s.grel = grads[1];
  s.dir[0] = ProjeDir{h, hr_t, noise_tail, p->De1, p->Dr1, p->bc1, grads[3], grads[4], grads[2]};
  s.dir[1] = ProjeDir{t, tr_h, noise_head, p->De2, p->Dr2, p->bc2, grads[6], grads[7], grads[5]};
  s.loss = loss; s.dbg_logit = dbg_logit; s.dbg_g = dbg_g;
  *loss = 0.f;
  int nd = 0;
  if (hr_t) s.dirs[nd++] = 0;
  if (tr_h) s.dirs[nd++] = 1;
  cuda_emu::launch(dim3((unsigned)B, (unsigned)nd), dim3(PROJE_THREADS), [&] { proje_step_kernel(s); });
}

void emu_labels_negatives(float* labels, int64_t B, int64_t N, const int64_t* neg, int64_t n_neg) {
  cuda_emu::launch(dim3((unsigned)B), dim3(128), [&] { proj_labels_neg_kernel(labels, N, neg, (int)n_neg); });
}

void emu_reg_l1(const float* const* w, float* const* g, const int64_t* n, int count, float lmbda, float* out) {
  L1Args a{};
  long long nmax = 0;
  for (int i = 0; i < count; ++i) {
    a.seg[i] = L1Seg{w[i], g ? g[i] : nullptr, (long long)n[i]};
    nmax = n[i] > nmax ? n[i] : nmax;
  }
  a.lmbda = lmbda; a.out = out;
  *out = 0.f;
  cuda_emu::launch(dim3(reg_l1_blocks(nmax, 2), (unsigned)count), dim3(256), [&] { reg_l1_kernel(a); });
}

}  // extern "C"
