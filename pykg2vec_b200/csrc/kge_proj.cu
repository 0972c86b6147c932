// kge_proj.cu — C-ABI launchers of the projection-model tail (kernels and launch plans:
// kge_proj.cuh), of the ConvE, HypER, InteractE and AcrE inference trunks (kge_conve.cuh, kge_hyper.cuh,
// kge_interacte.cuh, kge_acre.cuh, which reuse the same tiled GEMM — one translation unit so the kernel
// template is instantiated once), of ProjE_pointwise's trunk, training step and L1 regulariser
// (kge_proje.cuh), of TuckER's core matrices and trunk, forward and backward (kge_tucker.cuh) and of ConvE's,
// HypER's, InteractE's and AcrE's training-mode trunks, forward and backward (kge_conve_train.cuh,
// kge_hyper_train.cuh, kge_interacte_train.cuh, kge_acre_train.cuh).  Declarations and reference citations:
// include/kge_b200.h.
#include <cstdlib>

#include "kge_acre.cuh"
#include "kge_acre_train.cuh"
#include "kge_conve_train.cuh"
#include "kge_hyper_train.cuh"
#include "kge_interacte.cuh"
#include "kge_interacte_train.cuh"
#include "kge_proje.cuh"
#include "kge_tucker.cuh"

using namespace kge;

namespace {

int check_dims(const char* fn, int64_t B, int64_t N, int32_t k) {
  if (B < 0 || N < 0 || k <= 0 || B > (1ll << 30) || N > (1ll << 30)) {
    set_error("%s: bad shape B=%lld N=%lld k=%d", fn, (long long)B, (long long)N, (int)k);
    return KGE_EINVAL;
  }
  if ((B + PBM - 1) / PBM > 65535) {
    set_error("%s: %lld rows exceed 65535 row tiles per call", fn, (long long)B);
    return KGE_EINVAL;
  }
  return KGE_OK;
}

template <int EPI>
int launch_gemm(const ProjLaunch& L, cudaStream_t st, const char* what) {
  const dim3 grid(L.gx, L.gy, L.gz);
  switch (L.tile) {
    case PROJ_TILE_128x128: proj_gemm_kernel<EPI, 8, 8><<<grid, PTHREADS, 0, st>>>(L.g); break;
    case PROJ_TILE_64x128: proj_gemm_kernel<EPI, 4, 8><<<grid, PTHREADS, 0, st>>>(L.g); break;
    default: proj_gemm_kernel<EPI, 4, 4><<<grid, PTHREADS, 0, st>>>(L.g); break;
  }
  KGE_CHECK_LAUNCH(what);
  return KGE_OK;
}

// CTA tile of the forward / counting launches: proj_pick_tile(), or KGE_PROJ_TILE=0|1|2 in the
// environment (64x64 | 64x128 | 128x128; used by bench_proj.py and the tests to time / check each).
int pick_tile(int64_t M, int64_t N) {
  if (const char* e = getenv("KGE_PROJ_TILE"))
    if (e[0] >= '0' && e[0] <= '2' && e[1] == 0) return e[0] - '0';
  return proj_pick_tile(M, N, sm_count());
}

}  // namespace

extern "C" {

int kge_proj_tail_fwd(const float* x, const float* ent, const float* bias, int64_t B, int64_t N,
                      int32_t k, float* preds, void* stream) {
  if (!x || !ent || !preds) { set_error("kge_proj_tail_fwd: null pointer"); return KGE_EINVAL; }
  if (int rc = check_dims("kge_proj_tail_fwd", B, N, k)) return rc;
  if (B == 0 || N == 0) return KGE_OK;
  return launch_gemm<EPI_STORE>(proj_plan_fwd(x, ent, bias, B, N, k, preds, pick_tile(B, N)),
                                (cudaStream_t)stream, "proj_gemm_kernel<sigmoid>");
}

int kge_proj_tail_bwd(const float* grad_preds, const float* preds, const float* x, const float* ent,
                      int64_t B, int64_t N, int32_t k, float* grad_x, float* grad_ent,
                      float* grad_bias, void* stream) {
  if (!grad_preds || !preds || !x || !ent) { set_error("kge_proj_tail_bwd: null pointer"); return KGE_EINVAL; }
  if (int rc = check_dims("kge_proj_tail_bwd", B, N, k)) return rc;
  if ((N + PBM - 1) / PBM > 65535) { set_error("kge_proj_tail_bwd: N too large"); return KGE_EINVAL; }
  if (B == 0 || N == 0) return KGE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (grad_x)
    if (int rc = launch_gemm<EPI_ATOMIC>(proj_plan_grad_x(grad_preds, preds, ent, B, N, k, grad_x, 2 * sm_count()),
                                         st, "proj_gemm_kernel<grad_x>")) return rc;
  if (grad_ent)
    if (int rc = launch_gemm<EPI_ATOMIC>(proj_plan_grad_ent(grad_preds, preds, x, B, N, k, grad_ent), st,
                                         "proj_gemm_kernel<grad_ent>")) return rc;
  if (grad_bias) {
    proj_colsum_kernel<<<proj_tiles(N, 256), 256, 0, st>>>(grad_preds, preds, (int)B, N, grad_bias);
    KGE_CHECK_LAUNCH("proj_colsum_kernel");
  }
  return KGE_OK;
}

int kge_proj_bce(const float* preds, const float* labels, int64_t B, int64_t N, float label_scale,
                 float label_shift, float grad_scale, float* loss_out, float* grad_preds, void* stream) {
  if (!preds || !labels || !loss_out) { set_error("kge_proj_bce: null pointer"); return KGE_EINVAL; }
  if (B <= 0 || N <= 0) { set_error("kge_proj_bce: empty batch"); return KGE_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)B * N;
  KGE_CUDA_OK(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  proj_bce_kernel<<<proj_bce_blocks(n, sm_count()), 256, 0, st>>>(
      preds, labels, n, label_scale, label_shift, proj_bce_grad_factor(grad_scale, B, N),
      proj_bce_inv_count(B, N), loss_out, grad_preds);
  KGE_CHECK_LAUNCH("proj_bce_kernel");
  return KGE_OK;
}

int kge_proj_labels(const int64_t* rows, const int64_t* ptr, const int64_t* idx, int64_t B, int64_t N,
                    float* labels, void* stream) {
  if (!ptr || !idx || !labels) { set_error("kge_proj_labels: null pointer"); return KGE_EINVAL; }
  if (B < 0 || N <= 0 || B > 0x7fffffffll) { set_error("kge_proj_labels: bad shape"); return KGE_EINVAL; }
  if (B == 0) return KGE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  KGE_CUDA_OK(cudaMemsetAsync(labels, 0, sizeof(float) * (size_t)B * (size_t)N, st));
  proj_labels_kernel<<<(unsigned)B, 128, 0, st>>>(rows, ptr, idx, N, labels);
  KGE_CHECK_LAUNCH("proj_labels_kernel");
  return KGE_OK;
}

int64_t kge_proj_rank_workspace_bytes(int64_t Q) { return (Q > 0 ? Q : 1) * (int64_t)sizeof(float); }

int kge_proj_rank(const float* x, const float* ent, const float* bias, int64_t Q, int64_t N, int32_t k,
                  const int64_t* tgt, const int64_t* filt_ptr, const int64_t* filt_idx, int64_t filt_nnz,
                  int32_t direction, int32_t* counts, void* workspace, int64_t workspace_bytes,
                  void* stream) {
  if (!x || !ent || !tgt || !counts || !workspace) { set_error("kge_proj_rank: null pointer"); return KGE_EINVAL; }
  if (direction != 0 && direction != 1) { set_error("kge_proj_rank: direction must be 0 or 1"); return KGE_EINVAL; }
  if (int rc = check_dims("kge_proj_rank", Q, N, k)) return rc;
  if (workspace_bytes < kge_proj_rank_workspace_bytes(Q)) {
    set_error("kge_proj_rank: workspace too small");
    return KGE_EWORKSPACE;
  }
  if (Q == 0 || N == 0) return KGE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  float* thr = (float*)workspace;
  proj_target_kernel<<<proj_tiles(Q, 128), 128, 0, st>>>(x, ent, bias, tgt, (int)Q, k, thr);
  KGE_CHECK_LAUNCH("proj_target_kernel");
  if (int rc = launch_gemm<EPI_COUNT>(proj_plan_count(x, ent, bias, Q, N, k, thr, counts, direction,
                                                      pick_tile(Q, N)), st, "proj_gemm_kernel<count>")) return rc;
  if (filt_ptr && filt_idx && filt_nnz > 0) {
    proj_filter_kernel<<<(unsigned)Q, 128, 0, st>>>(x, ent, bias, tgt, filt_ptr, filt_idx, k, thr, counts,
                                                    2 * direction);
    KGE_CHECK_LAUNCH("proj_filter_kernel");
  }
  return KGE_OK;
}


// ---- ConvE inference trunk ----------------------------------------------------------------

int64_t kge_conve_trunk_workspace_bytes(const kge_conve_t* p, int64_t Q) {
  if (!p || p->hidden_size_1 < 3 || p->hidden_size < p->hidden_size_1) return 0;
  const int h2 = p->hidden_size / p->hidden_size_1;
  const long long F = conve_feat_width(h2, p->hidden_size_1), q = Q > 0 ? Q : 1;
  return (q * F + (long long)conve_fc_slices(F) * q * p->hidden_size) * (int64_t)sizeof(float);
}

int kge_conve_trunk_fwd(const kge_conve_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                        void* workspace, int64_t workspace_bytes, void* stream) {
  if (!p || !e || !r || !x || !workspace) { set_error("kge_conve_trunk_fwd: null pointer"); return KGE_EINVAL; }
  const int k = p->hidden_size, h1 = p->hidden_size_1;
  if (k <= 0 || h1 < 3 || k / h1 < 2 || (k / h1) * h1 != k || 2 * k > CONVE_MAX_IMAGE) {
    set_error("kge_conve_trunk_fwd: unsupported image (hidden_size %d, hidden_size_1 %d)", k, h1);
    return KGE_ENOTSUP;
  }
  const float* ptrs[] = {p->ent, p->rel, p->bn0_weight, p->bn0_bias, p->bn0_mean, p->bn0_var, p->conv_weight,
                         p->conv_bias, p->bn1_weight, p->bn1_bias, p->bn1_mean, p->bn1_var, p->fc_weight, p->fc_bias};
  for (const float* q : ptrs)
    if (!q) { set_error("kge_conve_trunk_fwd: null parameter tensor"); return KGE_EINVAL; }
  if (Q < 0 || (Q + PBM - 1) / PBM > 65535) { set_error("kge_conve_trunk_fwd: bad Q"); return KGE_EINVAL; }
  if (workspace_bytes < kge_conve_trunk_workspace_bytes(p, Q)) {
    set_error("kge_conve_trunk_fwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  if (Q == 0) return KGE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int h2 = k / h1;
  ConveFeat f{};
  f.ent = p->ent; f.rel = p->rel; f.e = e; f.r = r; f.k = k; f.h2 = h2; f.h1 = h1;
  f.bn0_w = p->bn0_weight; f.bn0_b = p->bn0_bias; f.bn0_mean = p->bn0_mean; f.bn0_var = p->bn0_var;
  f.bn0_eps = p->bn0_eps;
  f.conv_w = p->conv_weight; f.conv_b = p->conv_bias;
  f.bn1_w = p->bn1_weight; f.bn1_b = p->bn1_bias; f.bn1_mean = p->bn1_mean; f.bn1_var = p->bn1_var;
  f.bn1_eps = p->bn1_eps;
  f.feat = (float*)workspace;
  conve_feature_kernel<<<(unsigned)Q, CONVE_THREADS, 0, st>>>(f);
  KGE_CHECK_LAUNCH("conve_feature_kernel");
  const long long F = conve_feat_width(h2, h1);
  float* partial = f.feat + Q * F;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_fc(f.feat, p->fc_weight, Q, F, k, partial), st,
                                      "proj_gemm_kernel<fc>")) return rc;
  conve_fc_combine_kernel<<<proj_tiles(Q * k, 256), 256, 0, st>>>(partial, conve_fc_slices(F), Q * k, k,
                                                                 p->fc_bias, x);
  KGE_CHECK_LAUNCH("conve_fc_combine_kernel");
  return KGE_OK;
}


// ---- HypER inference trunk ----------------------------------------------------------------

static bool hyper_shape_ok(const kge_hyper_t* p) {
  return p && p->ent_hidden_size >= HYPER_FW && p->ent_hidden_size <= HYPER_MAX_DE && p->rel_hidden_size > 0 &&
         p->num_rel > 0;
}

int64_t kge_hyper_trunk_workspace_bytes(const kge_hyper_t* p, int64_t Q) {
  if (!hyper_shape_ok(p)) return 0;
  return hyper_layout(p->num_rel, Q > 0 ? Q : 1, p->ent_hidden_size).total * (int64_t)sizeof(float);
}

int kge_hyper_trunk_fwd(const kge_hyper_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                        void* workspace, int64_t workspace_bytes, void* stream) {
  if (!p || !workspace || (Q > 0 && (!e || !r || !x))) {   // an empty batch may pass null id / output pointers
    set_error("kge_hyper_trunk_fwd: null pointer");
    return KGE_EINVAL;
  }
  const int de = p->ent_hidden_size, dr = p->rel_hidden_size;
  if (de < HYPER_FW || de > HYPER_MAX_DE) {
    set_error("kge_hyper_trunk_fwd: unsupported ent_hidden_size %d (needs %d <= de <= %d)", de, HYPER_FW,
              HYPER_MAX_DE);
    return KGE_ENOTSUP;
  }
  if (dr <= 0 || p->num_rel <= 0 || (p->num_rel + PBM - 1) / PBM > 65535) {
    set_error("kge_hyper_trunk_fwd: bad rel_hidden_size %d / num_rel %lld", dr, (long long)p->num_rel);
    return KGE_EINVAL;
  }
  const float* ptrs[] = {p->ent, p->rel, p->bn0_weight, p->bn0_bias, p->bn0_mean, p->bn0_var, p->fc1_weight,
                         p->fc1_bias, p->bn1_weight, p->bn1_bias, p->bn1_mean, p->bn1_var, p->fc_weight, p->fc_bias,
                         p->bn2_weight, p->bn2_bias, p->bn2_mean, p->bn2_var};
  for (const float* t : ptrs)
    if (!t) { set_error("kge_hyper_trunk_fwd: null parameter tensor"); return KGE_EINVAL; }
  if (Q < 0 || (Q + PBM - 1) / PBM > 65535) { set_error("kge_hyper_trunk_fwd: bad Q"); return KGE_EINVAL; }
  if (workspace_bytes < kge_hyper_trunk_workspace_bytes(p, Q)) {
    set_error("kge_hyper_trunk_fwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  if (Q == 0) return KGE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const HyperLayout lay = hyper_layout(p->num_rel, Q, de);
  float* ws = (float*)workspace;
  if (int rc = launch_gemm<EPI_STORE>(hyper_plan_filters(p->rel, p->fc1_weight, p->fc1_bias, p->num_rel, dr,
                                                         ws + lay.filt), st, "proj_gemm_kernel<hyper filters>"))
    return rc;
  HyperFeat f{};
  f.ent = p->ent; f.filt = ws + lay.filt; f.e = e; f.r = r; f.de = de;
  f.bn0_w = p->bn0_weight; f.bn0_b = p->bn0_bias; f.bn0_mean = p->bn0_mean; f.bn0_var = p->bn0_var;
  f.bn0_eps = p->bn0_eps;
  f.bn1_w = p->bn1_weight; f.bn1_b = p->bn1_bias; f.bn1_mean = p->bn1_mean; f.bn1_var = p->bn1_var;
  f.bn1_eps = p->bn1_eps;
  f.feat = ws + lay.feat;
  hyper_feature_kernel<<<(unsigned)Q, HYPER_THREADS, 0, st>>>(f);
  KGE_CHECK_LAUNCH("hyper_feature_kernel");
  const long long F = hyper_feat_width(de);
  float* partial = ws + lay.partial;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_fc(f.feat, p->fc_weight, Q, F, de, partial), st,
                                      "proj_gemm_kernel<hyper fc>")) return rc;
  hyper_fc_combine_kernel<<<proj_tiles(Q * de, 256), 256, 0, st>>>(partial, conve_fc_slices(F), Q * de, de, p->fc_bias,
                                                                   p->bn2_weight, p->bn2_bias, p->bn2_mean,
                                                                   p->bn2_var, p->bn2_eps, x);
  KGE_CHECK_LAUNCH("hyper_fc_combine_kernel");
  return KGE_OK;
}


// ---- InteractE inference trunk ------------------------------------------------------------

// KGE_OK, or the error code of an unsupported / malformed geometry (message set for `fn`)
static int interacte_shape(const kge_interacte_t* p, const char* fn) {
  const int P = p->feature_permutation, F = p->num_filters, ks = p->kernel_size;
  const int H = 2 * p->reshape_width, W = p->reshape_height;
  if (P <= 0 || F <= 0 || ks <= 0 || p->reshape_width <= 0 || W <= 0 || p->num_rel <= 0 ||
      (long long)H * W > (1 << 20)) {
    set_error("%s: bad geometry P=%d F=%d ks=%d reshape %dx%d num_rel %lld", fn, P, F, ks, p->reshape_height,
              p->reshape_width, (long long)p->num_rel);
    return KGE_EINVAL;
  }
  if (ks < 3 || ks % 2 == 0 || ks / 2 > (H < W ? H : W)) {
    set_error("%s: unsupported kernel_size %d on a %dx%d image (needs an odd ks >= 3, ks/2 <= %d)", fn, ks, H, W,
              H < W ? H : W);
    return KGE_ENOTSUP;
  }
  const long long smem = interacte_smem(P, F, ks, H, W).total * (long long)sizeof(float);
  if (smem > INTERACTE_SMEM_MAX) {
    set_error("%s: filter bank + %d padded images need %lld bytes of shared memory (max %d)", fn, P, smem,
              INTERACTE_SMEM_MAX);
    return KGE_ENOTSUP;
  }
  const long long Fw = interacte_feat_width(P, F, H, W);
  if (Fw > (1ll << 30) || conve_fc_slices(Fw) > 65535) {
    set_error("%s: %lld features per query exceed the Linear layer's GEMM", fn, Fw);
    return KGE_ENOTSUP;
  }
  return KGE_OK;
}

int64_t kge_interacte_trunk_workspace_bytes(const kge_interacte_t* p, int64_t Q) {
  if (!p || interacte_shape(p, "kge_interacte_trunk_workspace_bytes")) return 0;
  return interacte_layout(Q > 0 ? Q : 1, p->feature_permutation, p->num_filters, 2 * p->reshape_width,
                          p->reshape_height).total * (int64_t)sizeof(float);
}

int kge_interacte_trunk_fwd(const kge_interacte_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                            void* workspace, int64_t workspace_bytes, void* stream) {
  if (!p || !workspace || (Q > 0 && (!e || !r || !x))) {   // an empty batch may pass null id / output pointers
    set_error("kge_interacte_trunk_fwd: null pointer");
    return KGE_EINVAL;
  }
  if (int rc = interacte_shape(p, "kge_interacte_trunk_fwd")) return rc;
  const float* ptrs[] = {p->ent, p->rel, p->bn0_weight, p->bn0_bias, p->bn0_mean, p->bn0_var, p->conv_filt,
                         p->bn1_weight, p->bn1_bias, p->bn1_mean, p->bn1_var, p->fc_weight, p->fc_bias,
                         p->bn2_weight, p->bn2_bias, p->bn2_mean, p->bn2_var};
  for (const float* t : ptrs)
    if (!t) { set_error("kge_interacte_trunk_fwd: null parameter tensor"); return KGE_EINVAL; }
  if (!p->perm) { set_error("kge_interacte_trunk_fwd: null perm"); return KGE_EINVAL; }
  if (Q < 0 || (Q + PBM - 1) / PBM > 65535) { set_error("kge_interacte_trunk_fwd: bad Q"); return KGE_EINVAL; }
  if (workspace_bytes < kge_interacte_trunk_workspace_bytes(p, Q)) {
    set_error("kge_interacte_trunk_fwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  if (Q == 0) return KGE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int P = p->feature_permutation, F = p->num_filters, ks = p->kernel_size;
  const int H = 2 * p->reshape_width, W = p->reshape_height, k = p->reshape_width * p->reshape_height;
  const InteracteLayout lay = interacte_layout(Q, P, F, H, W);
  float* ws = (float*)workspace;
  InteracteFeat f{};
  f.ent = p->ent; f.rel = p->rel; f.perm = p->perm; f.e = e; f.r = r;
  f.P = P; f.F = F; f.ks = ks; f.H = H; f.W = W;
  f.bn0_w = p->bn0_weight; f.bn0_b = p->bn0_bias; f.bn0_mean = p->bn0_mean; f.bn0_var = p->bn0_var;
  f.bn0_eps = p->bn0_eps;
  f.conv_filt = p->conv_filt;
  f.bn1_w = p->bn1_weight; f.bn1_b = p->bn1_bias; f.bn1_mean = p->bn1_mean; f.bn1_var = p->bn1_var;
  f.bn1_eps = p->bn1_eps;
  f.feat = ws + lay.feat;
  const size_t smem = (size_t)interacte_smem(P, F, ks, H, W).total * sizeof(float);
  if (smem > 48 * 1024)
    KGE_CUDA_OK(cudaFuncSetAttribute(interacte_feature_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem));
  interacte_feature_kernel<<<(unsigned)Q, INTERACTE_THREADS, smem, st>>>(f);
  KGE_CHECK_LAUNCH("interacte_feature_kernel");
  const long long Fw = interacte_feat_width(P, F, H, W);
  float* partial = ws + lay.partial;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_fc(f.feat, p->fc_weight, Q, Fw, k, partial), st,
                                      "proj_gemm_kernel<interacte fc>")) return rc;
  hyper_fc_combine_kernel<<<proj_tiles(Q * k, 256), 256, 0, st>>>(partial, conve_fc_slices(Fw), Q * k, k, p->fc_bias,
                                                                  p->bn2_weight, p->bn2_bias, p->bn2_mean,
                                                                  p->bn2_var, p->bn2_eps, x);
  KGE_CHECK_LAUNCH("hyper_fc_combine_kernel");
  return KGE_OK;
}


// ---- AcrE inference trunk -----------------------------------------------------------------

// KGE_OK, or the error code of an unsupported / malformed configuration (message set for `fn`)
static int acre_shape(const kge_acre_t* p, const char* fn) {
  const int C = p->in_channels;
  if ((p->way != 0 && p->way != 1) || C < 1 || p->first_atrous < 1 || p->second_atrous < 1 ||
      p->third_atrous < 1 || p->num_rel < 1) {
    set_error("%s: bad configuration way=%d in_channels=%d atrous %d/%d/%d num_rel %lld", fn, p->way, C,
              p->first_atrous, p->second_atrous, p->third_atrous, (long long)p->num_rel);
    return KGE_EINVAL;
  }
  if (p->hidden_size != ACRE_K) {
    set_error("%s: unsupported hidden_size %d (the trunk views each row as 10 x 20: needs 200)", fn,
              p->hidden_size);
    return KGE_ENOTSUP;
  }
  const long long smem = (p->way == 0 ? acre_serial_smem(C).total : acre_gate_smem(C)) * (long long)sizeof(float);
  if (smem > ACRE_SMEM_MAX) {
    set_error("%s: in_channels %d needs %lld bytes of shared memory in the %s way (max %d)", fn, C, smem,
              p->way == 0 ? "serial" : "parallel", ACRE_SMEM_MAX);
    return KGE_ENOTSUP;
  }
  return KGE_OK;
}

int64_t kge_acre_trunk_workspace_bytes(const kge_acre_t* p, int64_t Q) {
  if (!p || acre_shape(p, "kge_acre_trunk_workspace_bytes")) return 0;
  return acre_layout(Q > 0 ? Q : 1, p->in_channels, p->way == 1).total * (int64_t)sizeof(float);
}

int kge_acre_trunk_fwd(const kge_acre_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                       void* workspace, int64_t workspace_bytes, void* stream) {
  if (!p || !workspace || (Q > 0 && (!e || !r || !x))) {   // an empty batch may pass null id / output pointers
    set_error("kge_acre_trunk_fwd: null pointer");
    return KGE_EINVAL;
  }
  if (int rc = acre_shape(p, "kge_acre_trunk_fwd")) return rc;
  const bool par = p->way == 1;
  const float* ptrs[] = {p->ent, p->rel, p->bn0_weight, p->bn0_bias, p->bn0_mean, p->bn0_var, p->conv1_weight,
                         p->conv2_weight, p->conv3_weight, p->bn1_weight, p->bn1_bias, p->bn1_mean, p->bn1_var,
                         p->fc_weight, p->fc_bias, p->bn2_weight, p->bn2_bias, p->bn2_mean, p->bn2_var};
  for (const float* t : ptrs)
    if (!t) { set_error("kge_acre_trunk_fwd: null parameter tensor"); return KGE_EINVAL; }
  if (par && (!p->W_gate_e_weight || !p->W_gate_e_bias)) {
    set_error("kge_acre_trunk_fwd: the parallel way needs W_gate_e");
    return KGE_EINVAL;
  }
  const int nbias = (p->conv1_bias != nullptr) + (p->conv2_bias != nullptr) + (p->conv3_bias != nullptr);
  if (nbias != 0 && nbias != 3) {
    set_error("kge_acre_trunk_fwd: conv biases must be all set (acre_bias) or all NULL");
    return KGE_EINVAL;
  }
  const int C = p->in_channels;
  if (Q < 0 || (Q + PBM - 1) / PBM > 65535 || (par && (Q * C + PBM - 1) / PBM > 65535)) {
    set_error("kge_acre_trunk_fwd: bad Q %lld for in_channels %d", (long long)Q, C);
    return KGE_EINVAL;
  }
  if (workspace_bytes < kge_acre_trunk_workspace_bytes(p, Q)) {
    set_error("kge_acre_trunk_fwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  if (Q == 0) return KGE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const AcreLayout lay = acre_layout(Q, C, par);
  float* ws = (float*)workspace;
  AcreFeat f{};
  f.ent = p->ent; f.rel = p->rel; f.e = e; f.r = r; f.C = C;
  f.dil[0] = p->first_atrous; f.dil[1] = p->second_atrous; f.dil[2] = p->third_atrous;
  f.bn0_w = p->bn0_weight; f.bn0_b = p->bn0_bias; f.bn0_mean = p->bn0_mean; f.bn0_var = p->bn0_var;
  f.bn0_eps = p->bn0_eps;
  f.conv_w[0] = p->conv1_weight; f.conv_w[1] = p->conv2_weight; f.conv_w[2] = p->conv3_weight;
  f.conv_b[0] = p->conv1_bias; f.conv_b[1] = p->conv2_bias; f.conv_b[2] = p->conv3_bias;
  f.bn1_w = p->bn1_weight; f.bn1_b = p->bn1_bias; f.bn1_mean = p->bn1_mean; f.bn1_var = p->bn1_var;
  f.bn1_eps = p->bn1_eps;
  float* feat = ws + lay.feat;
  if (!par) {
    f.out = feat;
    const size_t smem = (size_t)acre_serial_smem(C).total * sizeof(float);
    if (smem > 48 * 1024)
      KGE_CUDA_OK(cudaFuncSetAttribute(acre_serial_feature_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
    acre_serial_feature_kernel<<<(unsigned)Q, ACRE_THREADS, smem, st>>>(f);
    KGE_CHECK_LAUNCH("acre_serial_feature_kernel");
  } else {
    f.out = ws + lay.gate;
    const size_t smem = (size_t)acre_gate_smem(C) * sizeof(float);
    if (smem > 48 * 1024)
      KGE_CUDA_OK(cudaFuncSetAttribute(acre_gate_input_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
    acre_gate_input_kernel<<<(unsigned)Q, ACRE_GATE_THREADS, smem, st>>>(f);
    KGE_CHECK_LAUNCH("acre_gate_input_kernel");
    const long long rows = Q * C;
    if (int rc = launch_gemm<EPI_STORE>(acre_plan_gate(f.out, p->W_gate_e_weight, p->W_gate_e_bias, rows, feat,
                                                       pick_tile(rows, ACRE_PIX)), st, "proj_gemm_kernel<acre gate>"))
      return rc;
    acre_bn1_relu_kernel<<<proj_tiles(rows * ACRE_PIX, 256), 256, 0, st>>>(feat, rows * ACRE_PIX, C, p->bn1_weight,
                                                                          p->bn1_bias, p->bn1_mean, p->bn1_var,
                                                                          p->bn1_eps);
    KGE_CHECK_LAUNCH("acre_bn1_relu_kernel");
  }
  const long long Fw = acre_feat_width(C);
  float* partial = ws + lay.partial;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_fc(feat, p->fc_weight, Q, Fw, ACRE_K, partial), st,
                                      "proj_gemm_kernel<acre fc>")) return rc;
  hyper_fc_combine_kernel<<<proj_tiles(Q * ACRE_K, 256), 256, 0, st>>>(partial, conve_fc_slices(Fw), Q * ACRE_K,
                                                                      ACRE_K, p->fc_bias, p->bn2_weight,
                                                                      p->bn2_bias, p->bn2_mean, p->bn2_var,
                                                                      p->bn2_eps, x);
  KGE_CHECK_LAUNCH("hyper_fc_combine_kernel");
  return KGE_OK;
}

// ---- ProjE_pointwise: trunk, fused training step, L1 regulariser, negative labels ----------

// KGE_OK, or the error code of a malformed / unsupported model struct (message set for `fn`)
static int proje_check(const kge_proje_t* p, const char* fn) {
  if (!p || !p->ent || !p->rel || !p->bc1 || !p->De1 || !p->Dr1 || !p->bc2 || !p->De2 || !p->Dr2) {
    set_error("%s: null pointer", fn);
    return KGE_EINVAL;
  }
  if (p->hidden_size <= 0 || p->num_ent <= 0 || p->num_ent > 0x7fffffffll || p->num_rel <= 0) {
    set_error("%s: bad shape hidden_size %d num_ent %lld num_rel %lld", fn, p->hidden_size,
              (long long)p->num_ent, (long long)p->num_rel);
    return KGE_EINVAL;
  }
  if (p->hidden_size > PROJE_MAX_K) {
    set_error("%s: hidden_size %d exceeds %d", fn, p->hidden_size, PROJE_MAX_K);
    return KGE_ENOTSUP;
  }
  return KGE_OK;
}

int kge_proje_trunk_fwd(const kge_proje_t* p, int32_t direction, const int64_t* e, const int64_t* r, int64_t Q,
                        const float* noise, float* x, void* stream) {
  if (int rc = proje_check(p, "kge_proje_trunk_fwd")) return rc;
  if (direction != 0 && direction != 1) { set_error("kge_proje_trunk_fwd: direction must be 0 or 1"); return KGE_EINVAL; }
  if (Q < 0 || Q > (1ll << 30) / p->hidden_size) { set_error("kge_proje_trunk_fwd: bad Q %lld", (long long)Q); return KGE_EINVAL; }
  if (Q == 0) return KGE_OK;
  if (!e || !r || !x) { set_error("kge_proje_trunk_fwd: null pointer"); return KGE_EINVAL; }
  const int k = p->hidden_size;
  const bool tail = direction == 0;
  proje_trunk_kernel<<<proj_tiles(Q * k, 256), 256, 0, (cudaStream_t)stream>>>(
      p->ent, p->rel, tail ? p->De1 : p->De2, tail ? p->Dr1 : p->Dr2, tail ? p->bc1 : p->bc2, e, r, Q, k, noise, x);
  KGE_CHECK_LAUNCH("proje_trunk_kernel");
  return KGE_OK;
}

int kge_proje_train_step(const kge_proje_t* p, const int64_t* h, const int64_t* r, const int64_t* t, int64_t B,
                         const float* hr_t, const float* tr_h, const float* noise_tail, const float* noise_head,
                         float* const* grads, float* loss_out, void* stream) {
  if (int rc = proje_check(p, "kge_proje_train_step")) return rc;
  if (!loss_out || !grads || (!hr_t && !tr_h)) {
    set_error("kge_proje_train_step: null loss_out / grads, or neither label matrix");
    return KGE_EINVAL;
  }
  if (B < 0 || B > 0x7fffffffll) { set_error("kge_proje_train_step: bad B %lld", (long long)B); return KGE_EINVAL; }
  cudaStream_t st = (cudaStream_t)stream;
  KGE_CUDA_OK(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  if (B == 0) return KGE_OK;
  if (!r || (hr_t && !h) || (tr_h && !t)) { set_error("kge_proje_train_step: null id pointer"); return KGE_EINVAL; }
  ProjeStep s{};
  s.ent = p->ent; s.rel = p->rel; s.r = r; s.N = p->num_ent; s.k = p->hidden_size; s.B = (int)B;
  s.gent = grads[0]; s.grel = grads[1];
  s.dir[0] = ProjeDir{h, hr_t, noise_tail, p->De1, p->Dr1, p->bc1, grads[3], grads[4], grads[2]};
  s.dir[1] = ProjeDir{t, tr_h, noise_head, p->De2, p->Dr2, p->bc2, grads[6], grads[7], grads[5]};
  s.loss = loss_out;
  int nd = 0;
  if (hr_t) s.dirs[nd++] = 0;
  if (tr_h) s.dirs[nd++] = 1;
  proje_step_kernel<<<dim3((unsigned)B, (unsigned)nd), PROJE_THREADS, 0, st>>>(s);
  KGE_CHECK_LAUNCH("proje_step_kernel");
  return KGE_OK;
}

int kge_reg_l1_dense(const float* const* w, float* const* grad, const int64_t* n, int32_t count, float lmbda,
                     float* reg_out, void* stream) {
  if (!w || !n || !reg_out || count < 0 || count > KGE_MAX_TABLES) {
    set_error("kge_reg_l1_dense: null pointer or bad count %d", (int)count);
    return KGE_EINVAL;
  }
  L1Args a{};
  long long nmax = 0;
  for (int i = 0; i < count; ++i) {
    if (n[i] < 0 || (n[i] > 0 && !w[i])) { set_error("kge_reg_l1_dense: bad tensor %d", i); return KGE_EINVAL; }
    a.seg[i] = L1Seg{w[i], grad ? grad[i] : nullptr, (long long)n[i]};
    if (n[i] > nmax) nmax = n[i];
  }
  a.lmbda = lmbda; a.out = reg_out;
  cudaStream_t st = (cudaStream_t)stream;
  KGE_CUDA_OK(cudaMemsetAsync(reg_out, 0, sizeof(float), st));
  if (count == 0 || nmax == 0) return KGE_OK;
  reg_l1_kernel<<<dim3(reg_l1_blocks(nmax, sm_count()), (unsigned)count), 256, 0, st>>>(a);
  KGE_CHECK_LAUNCH("reg_l1_kernel");
  return KGE_OK;
}

int kge_proj_labels_negatives(float* labels, int64_t B, int64_t N, const int64_t* neg, int64_t n_neg, void* stream) {
  if (B < 0 || N <= 0 || n_neg < 0 || n_neg > N || B > 0x7fffffffll) {
    set_error("kge_proj_labels_negatives: bad shape B=%lld N=%lld n_neg=%lld", (long long)B, (long long)N,
              (long long)n_neg);
    return KGE_EINVAL;
  }
  if (B == 0 || n_neg == 0) return KGE_OK;
  if (!labels || !neg) { set_error("kge_proj_labels_negatives: null pointer"); return KGE_EINVAL; }
  proj_labels_neg_kernel<<<(unsigned)B, 128, 0, (cudaStream_t)stream>>>(labels, N, neg, (int)n_neg);
  KGE_CHECK_LAUNCH("proj_labels_neg_kernel");
  return KGE_OK;
}

// ---- TuckER: core matrices per distinct relation, trunk forward / backward -----------------------

static int tucker_check(const kge_tucker_t* p, const char* fn) {
  if (!p || !p->ent || !p->rel || !p->W) { set_error("%s: null pointer", fn); return KGE_EINVAL; }
  if (p->d1 <= 0 || p->d2 <= 0 || p->num_ent <= 0 || p->num_rel <= 0) {
    set_error("%s: bad shape d1 %d d2 %d num_ent %lld num_rel %lld", fn, p->d1, p->d2, (long long)p->num_ent,
              (long long)p->num_rel);
    return KGE_EINVAL;
  }
  if (p->d1 > TUCKER_MAX_D || p->d2 > TUCKER_MAX_D) {
    set_error("%s: d1 %d / d2 %d exceed %d", fn, p->d1, p->d2, TUCKER_MAX_D);
    return KGE_ENOTSUP;
  }
  return KGE_OK;
}

// U core matrices per call: the GEMM's row-tile grid and 32-bit row count
static int tucker_check_U(int64_t U, const char* fn) {
  if (U < 0 || U > 65535ll * PBM) { set_error("%s: bad U %lld", fn, (long long)U); return KGE_EINVAL; }
  return KGE_OK;
}

static int tucker_mask(const kge_tucker_mask_t* m, const char* fn, TuckerMask* out) {
  *out = TuckerMask{};
  if (!m || m->mode == TUCKER_MASK_NONE) return KGE_OK;
  if (m->mode == TUCKER_MASK_EXPLICIT) {
    if (!m->noise1) { set_error("%s: explicit mask without noise1", fn); return KGE_EINVAL; }
    out->mode = TUCKER_MASK_EXPLICIT; out->noise1 = m->noise1;
    return KGE_OK;
  }
  if (m->mode != TUCKER_MASK_COUNTER || !(m->p >= 0.f)) { set_error("%s: bad mask mode %d / p", fn, m->mode); return KGE_EINVAL; }
  if (m->p == 0.f) return KGE_OK;   // nothing is dropped: no mask at all
  out->mode = TUCKER_MASK_COUNTER; out->seed = m->seed; out->offset = m->offset;
  tucker_mask_params(m->p, &out->thresh, &out->scale);
  return KGE_OK;
}

int64_t kge_tucker_workspace_bytes(const kge_tucker_t* p, int64_t U) {
  if (!p || p->d2 <= 0) return 0;
  return tucker_workspace_floats(U, p->d2) * (int64_t)sizeof(float);
}

int kge_tucker_cores(const kge_tucker_t* p, const int64_t* ids, int64_t U, float* M, void* workspace,
                     int64_t workspace_bytes, void* stream) {
  if (int rc = tucker_check(p, "kge_tucker_cores")) return rc;
  if (int rc = tucker_check_U(U, "kge_tucker_cores")) return rc;
  if (U == 0) return KGE_OK;
  if (!ids || !M || !workspace) { set_error("kge_tucker_cores: null pointer"); return KGE_EINVAL; }
  if (workspace_bytes < kge_tucker_workspace_bytes(p, U)) { set_error("kge_tucker_cores: workspace too small"); return KGE_EWORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  float* relU = (float*)workspace;
  tucker_gather_rows_kernel<<<proj_tiles(U * p->d2, 256), 256, 0, st>>>(p->rel, ids, U, p->d2, relU);
  KGE_CHECK_LAUNCH("tucker_gather_rows_kernel");
  return launch_gemm<EPI_STORE>(tucker_plan_cores(relU, p->W, U, p->d1, p->d2, M), st, "proj_gemm_kernel<tucker cores>");
}

static int tucker_trunk_args(const kge_tucker_t* p, const char* fn, const float* M, const int64_t* e,
                             const int64_t* slot, int64_t Q, const float* noise0, const kge_tucker_mask_t* mask,
                             const float* noise2, TuckerTrunk* a) {
  if (int rc = tucker_check(p, fn)) return rc;
  if (Q < 0 || Q > 0x7fffffffll) { set_error("%s: bad Q %lld", fn, (long long)Q); return KGE_EINVAL; }
  *a = TuckerTrunk{};
  if (int rc = tucker_mask(mask, fn, &a->mask)) return rc;
  if (Q == 0) return KGE_OK;
  if (!M || !e || !slot) { set_error("%s: null pointer", fn); return KGE_EINVAL; }
  a->ent = p->ent; a->M = M; a->e = e; a->slot = slot; a->d1 = p->d1; a->noise0 = noise0; a->noise2 = noise2;
  return KGE_OK;
}

int kge_tucker_trunk_fwd(const kge_tucker_t* p, const float* M, const int64_t* e, const int64_t* slot, int64_t Q,
                         const float* noise0, const kge_tucker_mask_t* mask, const float* noise2, float* x,
                         float* xpre, float* nrm, void* stream) {
  TuckerTrunk a;
  if (int rc = tucker_trunk_args(p, "kge_tucker_trunk_fwd", M, e, slot, Q, noise0, mask, noise2, &a)) return rc;
  if (Q == 0) return KGE_OK;
  if (!x || (!xpre != !nrm)) { set_error("kge_tucker_trunk_fwd: null x, or only one of xpre / nrm"); return KGE_EINVAL; }
  a.x = x; a.xpre = xpre; a.nrm = nrm;
  tucker_trunk_fwd_kernel<<<(unsigned)Q, TUCKER_THREADS, 0, (cudaStream_t)stream>>>(a);
  KGE_CHECK_LAUNCH("tucker_trunk_fwd_kernel");
  return KGE_OK;
}

int kge_tucker_trunk_bwd(const kge_tucker_t* p, const float* M, const int64_t* e, const int64_t* slot, int64_t Q,
                         const float* noise0, const kge_tucker_mask_t* mask, const float* noise2, const float* gx,
                         const float* xpre, const float* nrm, float* grad_ent, float* dM, void* stream) {
  TuckerTrunk a;
  if (int rc = tucker_trunk_args(p, "kge_tucker_trunk_bwd", M, e, slot, Q, noise0, mask, noise2, &a)) return rc;
  if (Q == 0 || (!grad_ent && !dM)) return KGE_OK;
  if (!gx || !xpre || !nrm) { set_error("kge_tucker_trunk_bwd: null pointer"); return KGE_EINVAL; }
  a.gx = gx; a.xpre = const_cast<float*>(xpre); a.nrm = const_cast<float*>(nrm); a.gent = grad_ent; a.dM = dM;
  tucker_trunk_bwd_kernel<<<(unsigned)Q, TUCKER_THREADS, 0, (cudaStream_t)stream>>>(a);
  KGE_CHECK_LAUNCH("tucker_trunk_bwd_kernel");
  return KGE_OK;
}

int kge_tucker_cores_bwd(const kge_tucker_t* p, const int64_t* ids, int64_t U, const float* dM, float* grad_rel,
                         float* grad_W, void* workspace, int64_t workspace_bytes, void* stream) {
  if (int rc = tucker_check(p, "kge_tucker_cores_bwd")) return rc;
  if (int rc = tucker_check_U(U, "kge_tucker_cores_bwd")) return rc;
  if (U == 0 || (!grad_rel && !grad_W)) return KGE_OK;
  if (!ids || !dM || !workspace) { set_error("kge_tucker_cores_bwd: null pointer"); return KGE_EINVAL; }
  if (workspace_bytes < kge_tucker_workspace_bytes(p, U)) { set_error("kge_tucker_cores_bwd: workspace too small"); return KGE_EWORKSPACE; }
  cudaStream_t st = (cudaStream_t)stream;
  const int d1 = p->d1, d2 = p->d2;
  float* relU = (float*)workspace;
  float* drelU = relU + (long long)U * d2;
  if (grad_W) {
    tucker_gather_rows_kernel<<<proj_tiles(U * d2, 256), 256, 0, st>>>(p->rel, ids, U, d2, relU);
    KGE_CHECK_LAUNCH("tucker_gather_rows_kernel");
    if (int rc = launch_gemm<EPI_ATOMIC>(tucker_plan_grad_W(relU, dM, U, d1, d2, grad_W), st,
                                         "proj_gemm_kernel<tucker grad_W>")) return rc;
  }
  if (grad_rel) {
    KGE_CUDA_OK(cudaMemsetAsync(drelU, 0, sizeof(float) * (size_t)U * d2, st));
    if (int rc = launch_gemm<EPI_ATOMIC>(tucker_plan_grad_rel(dM, p->W, U, d1, d2, drelU, 2 * sm_count()), st,
                                         "proj_gemm_kernel<tucker grad_rel>")) return rc;
    tucker_scatter_rows_kernel<<<proj_tiles(U * d2, 256), 256, 0, st>>>(drelU, ids, U, d2, grad_rel);
    KGE_CHECK_LAUNCH("tucker_scatter_rows_kernel");
  }
  return KGE_OK;
}

int kge_tucker_mask1(uint64_t seed, uint64_t offset, float p, int64_t Q, int32_t d1, float* out, void* stream) {
  if (Q < 0 || d1 <= 0 || d1 > TUCKER_MAX_D || !(p >= 0.f) || Q > (1ll << 40) / ((int64_t)d1 * d1)) {
    set_error("kge_tucker_mask1: bad shape / p");
    return KGE_EINVAL;
  }
  if (Q == 0) return KGE_OK;
  if (!out) { set_error("kge_tucker_mask1: null pointer"); return KGE_EINVAL; }
  TuckerMask m{};
  m.mode = TUCKER_MASK_COUNTER; m.seed = seed; m.offset = offset;
  tucker_mask_params(p, &m.thresh, &m.scale);
  if (p == 0.f) { m.thresh = 0u; m.scale = 1.0f; }
  const long long n = Q * (long long)d1 * d1;
  tucker_mask1_kernel<<<proj_tiles(n, 256), 256, 0, (cudaStream_t)stream>>>(m, n, out);
  KGE_CHECK_LAUNCH("tucker_mask1_kernel");
  return KGE_OK;
}

// ---- ConvE training-mode trunk: batch-statistics BatchNorm, dropout noise, forward and backward ----------------

// KGE_OK, or the error code of an unsupported image / malformed call (message set for `fn`)
static int conve_train_check(const kge_conve_train_t* p, const char* fn, int64_t Q, int64_t B) {
  if (!p) { set_error("%s: null pointer", fn); return KGE_EINVAL; }
  const int k = p->hidden_size, h1 = p->hidden_size_1;
  if (k <= 0 || h1 < 3 || k / h1 < 2 || (k / h1) * h1 != k || 2 * k > CONVE_MAX_IMAGE) {
    set_error("%s: unsupported image (hidden_size %d, hidden_size_1 %d)", fn, k, h1);
    return KGE_ENOTSUP;
  }
  const float* ptrs[] = {p->ent, p->rel, p->bn0_weight, p->bn0_bias, p->conv_weight, p->conv_bias, p->bn1_weight,
                         p->bn1_bias, p->fc_weight, p->fc_bias, p->bn2_weight, p->bn2_bias};
  for (const float* t : ptrs)
    if (!t) { set_error("%s: null parameter tensor", fn); return KGE_EINVAL; }
  const float* run[] = {p->bn0_mean, p->bn0_var, p->bn1_mean, p->bn1_var, p->bn2_mean, p->bn2_var};
  int nrun = 0;
  for (const float* t : run) nrun += t != nullptr;
  if (nrun != 0 && nrun != 6) { set_error("%s: running statistics must be all set or all NULL", fn); return KGE_EINVAL; }
  if (B < 2 || Q < B || Q % B != 0 || (Q + PBM - 1) / PBM > 65535 || Q > 0x7fffffffll) {
    set_error("%s: bad Q %lld / B %lld (Q a multiple of B >= 2)", fn, (long long)Q, (long long)B);
    return KGE_EINVAL;
  }
  return KGE_OK;
}

static ConveTrain conve_train_args(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q,
                                   int64_t B, const float* noise0, const float* noise1, const float* noise2,
                                   float* ws) {
  ConveTrain a{};
  a.ent = p->ent; a.rel = p->rel; a.e = e; a.r = r;
  a.k = p->hidden_size; a.h1 = p->hidden_size_1; a.h2 = a.k / a.h1; a.Q = Q; a.B = B;
  a.bn0_w = p->bn0_weight; a.bn0_b = p->bn0_bias; a.conv_w = p->conv_weight; a.conv_b = p->conv_bias;
  a.bn1_w = p->bn1_weight; a.bn1_b = p->bn1_bias; a.bn2_w = p->bn2_weight; a.bn2_b = p->bn2_bias;
  a.noise0 = noise0; a.noise1 = noise1; a.noise2 = noise2;
  const ConveTrainLayout L = conve_train_layout(Q, B, a.k, a.h1);
  a.img = ws + L.img; a.z1 = ws + L.z1; a.feat = ws + L.feat; a.hpre = ws + L.hpre;
  a.st0 = ws + L.st0; a.st1 = ws + L.st1; a.st2 = ws + L.st2; a.part0 = ws + L.part0; a.part1 = ws + L.part1;
  a.red0 = ws + L.red0; a.red1 = ws + L.red1; a.dz = ws + L.dz; a.dimg = ws + L.dimg; a.pw = ws + L.pw;
  a.pb = ws + L.pb;
  return a;
}

int64_t kge_conve_train_workspace_bytes(const kge_conve_train_t* p, int64_t Q, int64_t B) {
  if (!p || p->hidden_size_1 < 3 || p->hidden_size / p->hidden_size_1 < 2 || B < 1) return 0;
  const long long q = Q > B ? Q : B;
  return conve_train_layout(q, B, p->hidden_size, p->hidden_size_1).total * (int64_t)sizeof(float);
}

int kge_conve_train_fwd(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* noise0, const float* noise1, const float* noise2, float* x, void* workspace,
                        int64_t workspace_bytes, void* stream) {
  if (int rc = conve_train_check(p, "kge_conve_train_fwd", Q, B)) return rc;
  if (!e || !r || !x || !workspace) { set_error("kge_conve_train_fwd: null pointer"); return KGE_EINVAL; }
  if (workspace_bytes < kge_conve_train_workspace_bytes(p, Q, B)) {
    set_error("kge_conve_train_fwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const ConveTrain a = conve_train_args(p, e, r, Q, B, noise0, noise1, noise2, ws);
  const int k = a.k, plane = (2 * a.h2 - 2) * (a.h1 - 2);
  const long long F = conve_feat_width(a.h2, a.h1);
  conve_tr_gather_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("conve_tr_gather_kernel");
  conve_tr_bn_stats_kernel<<<1, 256, 0, st>>>(a.part0, Q, B, 1, (float)(2 * k), p->bn0_eps, p->bn0_momentum, a.st0,
                                              p->bn0_mean, p->bn0_var);
  KGE_CHECK_LAUNCH("conve_tr_bn_stats_kernel<bn0>");
  conve_tr_conv_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("conve_tr_conv_kernel");
  conve_tr_bn_stats_kernel<<<1, 256, 0, st>>>(a.part1, Q, B, CONVE_CH, (float)plane, p->bn1_eps, p->bn1_momentum,
                                              a.st1, p->bn1_mean, p->bn1_var);
  KGE_CHECK_LAUNCH("conve_tr_bn_stats_kernel<bn1>");
  conve_tr_feat_kernel<<<proj_tiles(Q * F, 256), 256, 0, st>>>(a, F, plane);
  KGE_CHECK_LAUNCH("conve_tr_feat_kernel");
  float* partial = ws + conve_train_layout(Q, B, k, a.h1).partial;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_fc(a.feat, p->fc_weight, Q, F, k, partial), st,
                                      "proj_gemm_kernel<conve train fc>")) return rc;
  conve_tr_fc_combine_kernel<<<proj_tiles(Q * k, 256), 256, 0, st>>>(partial, conve_fc_slices(F), Q * k, k, p->fc_bias,
                                                                    noise2, a.hpre);
  KGE_CHECK_LAUNCH("conve_tr_fc_combine_kernel");
  conve_tr_bn2_kernel<<<proj_tiles(k, 256), 256, 0, st>>>(a, p->bn2_eps, p->bn2_momentum, p->bn2_mean, p->bn2_var, x);
  KGE_CHECK_LAUNCH("conve_tr_bn2_kernel");
  return KGE_OK;
}

int kge_conve_train_bwd(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* noise0, const float* noise1, const float* noise2, const float* gx,
                        const float* x, float* const* grads, void* workspace, int64_t workspace_bytes, void* stream) {
  if (int rc = conve_train_check(p, "kge_conve_train_bwd", Q, B)) return rc;
  if (!e || !r || !gx || !x || !grads || !workspace) { set_error("kge_conve_train_bwd: null pointer"); return KGE_EINVAL; }
  for (int i = 0; i < KGE_CONVE_TRAIN_GRADS; ++i)
    if (!grads[i]) { set_error("kge_conve_train_bwd: null gradient buffer %d", i); return KGE_EINVAL; }
  if (workspace_bytes < kge_conve_train_workspace_bytes(p, Q, B)) {
    set_error("kge_conve_train_bwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const ConveTrain a = conve_train_args(p, e, r, Q, B, noise0, noise1, noise2, ws);
  const int k = a.k;
  const long long F = conve_feat_width(a.h2, a.h1);
  float* dh = ws + conve_train_layout(Q, B, k, a.h1).dh;
  // grads: ent, rel, bn0.w, bn0.b, conv.w, conv.b, bn1.w, bn1.b, fc.w, fc.b, bn2.w, bn2.b
  conve_tr_bn2_bwd_kernel<<<proj_tiles(k, 256), 256, 0, st>>>(a, gx, x, dh, grads[10], grads[11], grads[9]);
  KGE_CHECK_LAUNCH("conve_tr_bn2_bwd_kernel");
  if (int rc = launch_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(dh, a.feat, Q, F, k, grads[8]), st,
                                       "proj_gemm_kernel<conve grad fc_w>")) return rc;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_grad_feat(dh, p->fc_weight, Q, F, k, a.dz), st,
                                      "proj_gemm_kernel<conve grad feat>")) return rc;
  conve_tr_bn1_bwd_part_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("conve_tr_bn1_bwd_part_kernel");
  conve_tr_reduce_kernel<<<1, 256, 0, st>>>(a.part1, Q, B, CONVE_CH, a.red1, grads[6], grads[7]);
  KGE_CHECK_LAUNCH("conve_tr_reduce_kernel<bn1>");
  conve_tr_conv_bwd_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("conve_tr_conv_bwd_kernel");
  conve_tr_colsum_kernel<<<proj_tiles(CONVE_TAPS, 256), 256, 0, st>>>(a.pw, Q, CONVE_TAPS, grads[4]);
  KGE_CHECK_LAUNCH("conve_tr_colsum_kernel<conv weight>");
  conve_tr_colsum_kernel<<<1, 256, 0, st>>>(a.pb, Q, CONVE_CH, grads[5]);
  KGE_CHECK_LAUNCH("conve_tr_colsum_kernel<conv bias>");
  conve_tr_reduce_kernel<<<1, 256, 0, st>>>(a.part0, Q, B, 1, a.red0, grads[2], grads[3]);
  KGE_CHECK_LAUNCH("conve_tr_reduce_kernel<bn0>");
  conve_tr_bn0_bwd_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a, grads[0], grads[1]);
  KGE_CHECK_LAUNCH("conve_tr_bn0_bwd_kernel");
  return KGE_OK;
}

// ---- HypER training-mode trunk: relation-generated filters, batch-statistics BatchNorm, forward and backward ------

// KGE_OK, or the error code of an unsupported width / malformed call (message set for `fn`)
static int hyper_train_check(const kge_hyper_train_t* p, const char* fn, int64_t Q, int64_t B) {
  if (!p) { set_error("%s: null pointer", fn); return KGE_EINVAL; }
  const int de = p->ent_hidden_size, dr = p->rel_hidden_size;
  if (de < HYPER_FW || de > HYPER_MAX_DE) {
    set_error("%s: unsupported ent_hidden_size %d (needs %d <= de <= %d)", fn, de, HYPER_FW, HYPER_MAX_DE);
    return KGE_ENOTSUP;
  }
  if (dr <= 0 || dr > (1 << 20)) { set_error("%s: bad rel_hidden_size %d", fn, dr); return KGE_EINVAL; }
  const float* ptrs[] = {p->ent, p->rel, p->bn0_weight, p->bn0_bias, p->bn1_weight, p->bn1_bias, p->fc_weight,
                         p->fc_bias, p->bn2_weight, p->bn2_bias, p->fc1_weight, p->fc1_bias};
  for (const float* t : ptrs)
    if (!t) { set_error("%s: null parameter tensor", fn); return KGE_EINVAL; }
  const float* run[] = {p->bn0_mean, p->bn0_var, p->bn1_mean, p->bn1_var, p->bn2_mean, p->bn2_var};
  int nrun = 0;
  for (const float* t : run) nrun += t != nullptr;
  if (nrun != 0 && nrun != 6) { set_error("%s: running statistics must be all set or all NULL", fn); return KGE_EINVAL; }
  if (B < 2 || Q < B || Q % B != 0 || (Q + PBM - 1) / PBM > 65535 || Q > 0x7fffffffll) {
    set_error("%s: bad Q %lld / B %lld (Q a multiple of B >= 2)", fn, (long long)Q, (long long)B);
    return KGE_EINVAL;
  }
  return KGE_OK;
}

static HyperTrain hyper_train_args(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q,
                                   int64_t B, const float* noise0, const float* noise1, const float* noise2,
                                   float* ws) {
  HyperTrain a{};
  a.ent = p->ent; a.e = e; a.r = r;
  a.de = p->ent_hidden_size; a.dr = p->rel_hidden_size; a.Q = Q; a.B = B;
  a.ent_pad = p->ent_padding_idx; a.rel_pad = p->rel_padding_idx;
  a.bn0_w = p->bn0_weight; a.bn0_b = p->bn0_bias; a.bn1_w = p->bn1_weight; a.bn1_b = p->bn1_bias;
  a.bn2_w = p->bn2_weight; a.bn2_b = p->bn2_bias;
  a.noise0 = noise0; a.noise1 = noise1; a.noise2 = noise2;
  const HyperTrainLayout L = hyper_train_layout(Q, B, a.de, a.dr);
  a.relr = ws + L.relr; a.filt = ws + L.filt; a.img = ws + L.img; a.z1 = ws + L.z1; a.feat = ws + L.feat;
  a.hpre = ws + L.hpre; a.st0 = ws + L.st0; a.st1 = ws + L.st1; a.st2 = ws + L.st2; a.part0 = ws + L.part0;
  a.part1 = ws + L.part1; a.red0 = ws + L.red0; a.red1 = ws + L.red1; a.dh = ws + L.dh; a.dz = ws + L.dz;
  a.dimg = ws + L.dimg; a.dw = ws + L.dw; a.drel = ws + L.drel;
  return a;
}

int64_t kge_hyper_train_workspace_bytes(const kge_hyper_train_t* p, int64_t Q, int64_t B) {
  if (!p || p->ent_hidden_size < HYPER_FW || p->ent_hidden_size > HYPER_MAX_DE || p->rel_hidden_size <= 0 || B < 1)
    return 0;
  const long long q = Q > B ? Q : B;
  return hyper_train_layout(q, B, p->ent_hidden_size, p->rel_hidden_size).total * (int64_t)sizeof(float);
}

int kge_hyper_train_fwd(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* noise0, const float* noise1, const float* noise2, float* x, void* workspace,
                        int64_t workspace_bytes, void* stream) {
  if (int rc = hyper_train_check(p, "kge_hyper_train_fwd", Q, B)) return rc;
  if (!e || !r || !x || !workspace) { set_error("kge_hyper_train_fwd: null pointer"); return KGE_EINVAL; }
  if (workspace_bytes < kge_hyper_train_workspace_bytes(p, Q, B)) {
    set_error("kge_hyper_train_fwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const HyperTrain a = hyper_train_args(p, e, r, Q, B, noise0, noise1, noise2, ws);
  const int de = a.de, dr = a.dr, Wo = de - HYPER_FW + 1;
  const long long F = hyper_feat_width(de);
  tucker_gather_rows_kernel<<<proj_tiles(Q * dr, 256), 256, 0, st>>>(p->rel, r, Q, dr, a.relr);
  KGE_CHECK_LAUNCH("tucker_gather_rows_kernel<hyper rel>");
  if (int rc = launch_gemm<EPI_STORE>(hyper_plan_filters(a.relr, p->fc1_weight, p->fc1_bias, Q, dr, a.filt), st,
                                      "proj_gemm_kernel<hyper train filters>")) return rc;
  hyper_tr_gather_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("hyper_tr_gather_kernel");
  conve_tr_bn_stats_kernel<<<1, 256, 0, st>>>(a.part0, Q, B, 1, (float)de, p->bn0_eps, p->bn0_momentum, a.st0,
                                              p->bn0_mean, p->bn0_var);
  KGE_CHECK_LAUNCH("conve_tr_bn_stats_kernel<hyper bn0>");
  hyper_tr_conv_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("hyper_tr_conv_kernel");
  conve_tr_bn_stats_kernel<<<1, 256, 0, st>>>(a.part1, Q, B, HYPER_CH, (float)Wo, p->bn1_eps, p->bn1_momentum,
                                              a.st1, p->bn1_mean, p->bn1_var);
  KGE_CHECK_LAUNCH("conve_tr_bn_stats_kernel<hyper bn1>");
  hyper_tr_feat_kernel<<<proj_tiles(Q * F, 256), 256, 0, st>>>(a, F, Wo);
  KGE_CHECK_LAUNCH("hyper_tr_feat_kernel");
  float* partial = ws + hyper_train_layout(Q, B, de, dr).partial;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_fc(a.feat, p->fc_weight, Q, F, de, partial), st,
                                      "proj_gemm_kernel<hyper train fc>")) return rc;
  conve_tr_fc_combine_kernel<<<proj_tiles(Q * de, 256), 256, 0, st>>>(partial, conve_fc_slices(F), Q * de, de,
                                                                     p->fc_bias, noise2, a.hpre);
  KGE_CHECK_LAUNCH("conve_tr_fc_combine_kernel<hyper>");
  conve_tr_bn2_kernel<<<proj_tiles(de, 256), 256, 0, st>>>(hyper_tr_bn2_view(a), p->bn2_eps, p->bn2_momentum,
                                                           p->bn2_mean, p->bn2_var, x);
  KGE_CHECK_LAUNCH("conve_tr_bn2_kernel<hyper>");
  return KGE_OK;
}

int kge_hyper_train_bwd(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* noise0, const float* noise1, const float* noise2, const float* gx,
                        const float* x, float* const* grads, void* workspace, int64_t workspace_bytes, void* stream) {
  if (int rc = hyper_train_check(p, "kge_hyper_train_bwd", Q, B)) return rc;
  if (!e || !r || !gx || !x || !grads || !workspace) { set_error("kge_hyper_train_bwd: null pointer"); return KGE_EINVAL; }
  for (int i = 0; i < KGE_HYPER_TRAIN_GRADS; ++i)
    if (!grads[i]) { set_error("kge_hyper_train_bwd: null gradient buffer %d", i); return KGE_EINVAL; }
  if (workspace_bytes < kge_hyper_train_workspace_bytes(p, Q, B)) {
    set_error("kge_hyper_train_bwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const HyperTrain a = hyper_train_args(p, e, r, Q, B, noise0, noise1, noise2, ws);
  const int de = a.de, dr = a.dr;
  const long long F = hyper_feat_width(de);
  // grads: ent, rel, bn0.w, bn0.b, bn1.w, bn1.b, fc.w, fc.b, bn2.w, bn2.b, fc1.w, fc1.b
  conve_tr_bn2_bwd_kernel<<<proj_tiles(de, 256), 256, 0, st>>>(hyper_tr_bn2_view(a), gx, x, a.dh, grads[8], grads[9],
                                                               grads[7]);
  KGE_CHECK_LAUNCH("conve_tr_bn2_bwd_kernel<hyper>");
  if (int rc = launch_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(a.dh, a.feat, Q, F, de, grads[6]), st,
                                       "proj_gemm_kernel<hyper grad fc_w>")) return rc;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_grad_feat(a.dh, p->fc_weight, Q, F, de, a.dz), st,
                                      "proj_gemm_kernel<hyper grad feat>")) return rc;
  hyper_tr_bn1_bwd_part_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("hyper_tr_bn1_bwd_part_kernel");
  conve_tr_reduce_kernel<<<1, 256, 0, st>>>(a.part1, Q, B, HYPER_CH, a.red1, grads[4], grads[5]);
  KGE_CHECK_LAUNCH("conve_tr_reduce_kernel<hyper bn1>");
  hyper_tr_conv_bwd_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("hyper_tr_conv_bwd_kernel");
  conve_tr_reduce_kernel<<<1, 256, 0, st>>>(a.part0, Q, B, 1, a.red0, grads[2], grads[3]);
  KGE_CHECK_LAUNCH("conve_tr_reduce_kernel<hyper bn0>");
  hyper_tr_bn0_bwd_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a, grads[0]);
  KGE_CHECK_LAUNCH("hyper_tr_bn0_bwd_kernel");
  if (int rc = launch_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(a.dw, a.relr, Q, dr, HYPER_FILT, grads[10]), st,
                                       "proj_gemm_kernel<hyper grad fc1_w>")) return rc;
  conve_tr_colsum_kernel<<<proj_tiles(HYPER_FILT, 256), 256, 0, st>>>(a.dw, Q, HYPER_FILT, grads[11]);
  KGE_CHECK_LAUNCH("conve_tr_colsum_kernel<hyper fc1 bias>");
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_grad_feat(a.dw, p->fc1_weight, Q, dr, HYPER_FILT, a.drel), st,
                                      "proj_gemm_kernel<hyper grad rel>")) return rc;
  hyper_tr_scatter_rel_kernel<<<proj_tiles(Q * dr, 256), 256, 0, st>>>(a.drel, r, Q, dr, a.rel_pad, grads[1]);
  KGE_CHECK_LAUNCH("hyper_tr_scatter_rel_kernel");
  return KGE_OK;
}

// ---- InteractE training-mode trunk: chequer-permuted circular convolution, batch-statistics BatchNorm -------------

// KGE_OK, or the error code of an unsupported geometry / malformed call (message set for `fn`)
static int interacte_train_check(const kge_interacte_train_t* p, const char* fn, int64_t Q, int64_t B) {
  if (!p) { set_error("%s: null pointer", fn); return KGE_EINVAL; }
  kge_interacte_t geo{};   // the inference trunk's shape rules
  geo.feature_permutation = p->feature_permutation; geo.num_filters = p->num_filters;
  geo.kernel_size = p->kernel_size; geo.reshape_height = p->reshape_height; geo.reshape_width = p->reshape_width;
  geo.num_rel = 1;
  if (int rc = interacte_shape(&geo, fn)) return rc;
  const float* ptrs[] = {p->ent, p->rel, p->bn0_weight, p->bn0_bias, p->conv_filt, p->bn1_weight, p->bn1_bias,
                         p->fc_weight, p->fc_bias, p->bn2_weight, p->bn2_bias};
  for (const float* t : ptrs)
    if (!t) { set_error("%s: null parameter tensor", fn); return KGE_EINVAL; }
  if (!p->perm) { set_error("%s: null perm", fn); return KGE_EINVAL; }
  const float* run[] = {p->bn0_mean, p->bn0_var, p->bn1_mean, p->bn1_var, p->bn2_mean, p->bn2_var};
  int nrun = 0;
  for (const float* t : run) nrun += t != nullptr;
  if (nrun != 0 && nrun != 6) { set_error("%s: running statistics must be all set or all NULL", fn); return KGE_EINVAL; }
  if (B < 2 || Q < B || Q % B != 0 || (Q + PBM - 1) / PBM > 65535 || Q > 0x7fffffffll) {
    set_error("%s: bad Q %lld / B %lld (Q a multiple of B >= 2)", fn, (long long)Q, (long long)B);
    return KGE_EINVAL;
  }
  return KGE_OK;
}

static InteracteTrainLayout interacte_train_layout_of(const kge_interacte_train_t* p, int64_t Q, int64_t B) {
  return interacte_train_layout(Q, B, p->feature_permutation, p->num_filters, p->kernel_size, 2 * p->reshape_width,
                                p->reshape_height);
}

static InteracteTrain interacte_train_args(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r,
                                           int64_t Q, int64_t B, const float* noise0, const float* noise1,
                                           const float* noise2, float* ws) {
  InteracteTrain a{};
  a.ent = p->ent; a.rel = p->rel; a.perm = p->perm; a.e = e; a.r = r;
  a.P = p->feature_permutation; a.F = p->num_filters; a.ks = p->kernel_size;
  a.H = 2 * p->reshape_width; a.W = p->reshape_height; a.Q = Q; a.B = B;
  a.bn0_w = p->bn0_weight; a.bn0_b = p->bn0_bias; a.filt = p->conv_filt; a.bn1_w = p->bn1_weight;
  a.bn1_b = p->bn1_bias; a.bn2_w = p->bn2_weight; a.bn2_b = p->bn2_bias;
  a.noise0 = noise0; a.noise1 = noise1; a.noise2 = noise2;
  const InteracteTrainLayout L = interacte_train_layout_of(p, Q, B);
  a.img = ws + L.img; a.z1 = ws + L.z1; a.feat = ws + L.feat; a.hpre = ws + L.hpre; a.st0 = ws + L.st0;
  a.st1 = ws + L.st1; a.st2 = ws + L.st2; a.part0 = ws + L.part0; a.part1 = ws + L.part1; a.red0 = ws + L.red0;
  a.red1 = ws + L.red1; a.dh = ws + L.dh; a.dimg = ws + L.dimg; a.pw = ws + L.pw;
  return a;
}

// dynamic shared memory of a launch above the 48 KB default: opt the kernel in first
static int interacte_tr_smem_optin(const void* kernel, size_t bytes) {
  if (bytes > 48 * 1024) KGE_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return KGE_OK;
}

int64_t kge_interacte_train_workspace_bytes(const kge_interacte_train_t* p, int64_t Q, int64_t B) {
  if (!p || B < 1) return 0;
  kge_interacte_t geo{};
  geo.feature_permutation = p->feature_permutation; geo.num_filters = p->num_filters;
  geo.kernel_size = p->kernel_size; geo.reshape_height = p->reshape_height; geo.reshape_width = p->reshape_width;
  geo.num_rel = 1;
  if (interacte_shape(&geo, "kge_interacte_train_workspace_bytes")) return 0;
  return interacte_train_layout_of(p, Q > B ? Q : B, B).total * (int64_t)sizeof(float);
}

int kge_interacte_train_fwd(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                            const float* noise0, const float* noise1, const float* noise2, float* x, void* workspace,
                            int64_t workspace_bytes, void* stream) {
  if (int rc = interacte_train_check(p, "kge_interacte_train_fwd", Q, B)) return rc;
  if (!e || !r || !x || !workspace) { set_error("kge_interacte_train_fwd: null pointer"); return KGE_EINVAL; }
  if (workspace_bytes < kge_interacte_train_workspace_bytes(p, Q, B)) {
    set_error("kge_interacte_train_fwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const InteracteTrain a = interacte_train_args(p, e, r, Q, B, noise0, noise1, noise2, ws);
  const int P = a.P, F = a.F, HW = a.H * a.W, k = HW / 2, C1 = P * F;
  const long long Fw = (long long)C1 * HW;
  interacte_tr_gather_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("interacte_tr_gather_kernel");
  conve_tr_bn_stats_kernel<<<proj_tiles(P, 256), 256, 0, st>>>(a.part0, Q, B, P, (float)HW, p->bn0_eps,
                                                              p->bn0_momentum, a.st0, p->bn0_mean, p->bn0_var);
  KGE_CHECK_LAUNCH("conve_tr_bn_stats_kernel<interacte bn0>");
  const size_t smem = (size_t)interacte_train_smem(P, F, a.ks, a.H, a.W).total * sizeof(float);
  if (int rc = interacte_tr_smem_optin((const void*)interacte_tr_conv_kernel, smem)) return rc;
  interacte_tr_conv_kernel<<<(unsigned)Q, CONVE_TR_THREADS, smem, st>>>(a);
  KGE_CHECK_LAUNCH("interacte_tr_conv_kernel");
  conve_tr_bn_stats_kernel<<<proj_tiles(C1, 256), 256, 0, st>>>(a.part1, Q, B, C1, (float)HW, p->bn1_eps,
                                                               p->bn1_momentum, a.st1, p->bn1_mean, p->bn1_var);
  KGE_CHECK_LAUNCH("conve_tr_bn_stats_kernel<interacte bn1>");
  interacte_tr_feat_kernel<<<proj_tiles(Q * Fw, 256), 256, 0, st>>>(a, Fw, HW);
  KGE_CHECK_LAUNCH("interacte_tr_feat_kernel");
  float* partial = ws + interacte_train_layout_of(p, Q, B).partial;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_fc(a.feat, p->fc_weight, Q, Fw, k, partial), st,
                                      "proj_gemm_kernel<interacte train fc>")) return rc;
  conve_tr_fc_combine_kernel<<<proj_tiles(Q * k, 256), 256, 0, st>>>(partial, conve_fc_slices(Fw), Q * k, k,
                                                                    p->fc_bias, noise2, a.hpre);
  KGE_CHECK_LAUNCH("conve_tr_fc_combine_kernel<interacte>");
  conve_tr_bn2_kernel<<<proj_tiles(k, 256), 256, 0, st>>>(interacte_tr_bn2_view(a), p->bn2_eps, p->bn2_momentum,
                                                          p->bn2_mean, p->bn2_var, x);
  KGE_CHECK_LAUNCH("conve_tr_bn2_kernel<interacte>");
  return KGE_OK;
}

int kge_interacte_train_bwd(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                            const float* noise0, const float* noise1, const float* noise2, const float* gx,
                            const float* x, float* const* grads, void* workspace, int64_t workspace_bytes,
                            void* stream) {
  if (int rc = interacte_train_check(p, "kge_interacte_train_bwd", Q, B)) return rc;
  if (!e || !r || !gx || !x || !grads || !workspace) {
    set_error("kge_interacte_train_bwd: null pointer");
    return KGE_EINVAL;
  }
  for (int i = 0; i < KGE_INTERACTE_TRAIN_GRADS; ++i)
    if (!grads[i]) { set_error("kge_interacte_train_bwd: null gradient buffer %d", i); return KGE_EINVAL; }
  if (workspace_bytes < kge_interacte_train_workspace_bytes(p, Q, B)) {
    set_error("kge_interacte_train_bwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const InteracteTrain a = interacte_train_args(p, e, r, Q, B, noise0, noise1, noise2, ws);
  const int P = a.P, F = a.F, HW = a.H * a.W, k = HW / 2, C1 = P * F, taps = a.ks * a.ks;
  const long long Fw = (long long)C1 * HW;
  // grads: ent, rel, bn0.w, bn0.b, conv_filt, bn1.w, bn1.b, fc.w, fc.b, bn2.w, bn2.b
  conve_tr_bn2_bwd_kernel<<<proj_tiles(k, 256), 256, 0, st>>>(interacte_tr_bn2_view(a), gx, x, a.dh, grads[9],
                                                              grads[10], grads[8]);
  KGE_CHECK_LAUNCH("conve_tr_bn2_bwd_kernel<interacte>");
  // d fc.weight reads feat before d feat overwrites it (same stream, in order)
  if (int rc = launch_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(a.dh, a.feat, Q, Fw, k, grads[7]), st,
                                       "proj_gemm_kernel<interacte grad fc_w>")) return rc;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_grad_feat(a.dh, p->fc_weight, Q, Fw, k, a.feat), st,
                                      "proj_gemm_kernel<interacte grad feat>")) return rc;
  interacte_tr_bn1_bwd_part_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("interacte_tr_bn1_bwd_part_kernel");
  conve_tr_reduce_kernel<<<proj_tiles(C1, 256), 256, 0, st>>>(a.part1, Q, B, C1, a.red1, grads[5], grads[6]);
  KGE_CHECK_LAUNCH("conve_tr_reduce_kernel<interacte bn1>");
  const size_t smem = (size_t)interacte_train_smem(P, F, a.ks, a.H, a.W).total * sizeof(float);
  if (int rc = interacte_tr_smem_optin((const void*)interacte_tr_conv_bwd_kernel, smem)) return rc;
  interacte_tr_conv_bwd_kernel<<<(unsigned)Q, CONVE_TR_THREADS, smem, st>>>(a);
  KGE_CHECK_LAUNCH("interacte_tr_conv_bwd_kernel");
  conve_tr_colsum_kernel<<<proj_tiles(F * taps, 256), 256, 0, st>>>(a.pw, Q, F * taps, grads[4]);
  KGE_CHECK_LAUNCH("conve_tr_colsum_kernel<interacte conv_filt>");
  conve_tr_reduce_kernel<<<proj_tiles(P, 256), 256, 0, st>>>(a.part0, Q, B, P, a.red0, grads[2], grads[3]);
  KGE_CHECK_LAUNCH("conve_tr_reduce_kernel<interacte bn0>");
  const size_t ismem = (size_t)P * HW * sizeof(int);
  if (int rc = interacte_tr_smem_optin((const void*)interacte_tr_bn0_bwd_kernel, ismem)) return rc;
  interacte_tr_bn0_bwd_kernel<<<(unsigned)Q, CONVE_TR_THREADS, ismem, st>>>(a, grads[0], grads[1]);
  KGE_CHECK_LAUNCH("interacte_tr_bn0_bwd_kernel");
  return KGE_OK;
}

// ---- AcrE training-mode trunk: serial / parallel atrous convolutions, batch-statistics BatchNorm ------------------

// KGE_OK, or the error code of an unsupported configuration (message set for `fn`); the shape rules only
static int acre_train_shape(const kge_acre_train_t* p, const char* fn) {
  const int C = p->in_channels;
  if ((p->way != 0 && p->way != 1) || C < 1 || p->first_atrous < 1 || p->second_atrous < 1 || p->third_atrous < 1 ||
      p->num_rel < 1) {
    set_error("%s: bad configuration way=%d in_channels=%d atrous %d/%d/%d num_rel %lld", fn, p->way, C,
              p->first_atrous, p->second_atrous, p->third_atrous, (long long)p->num_rel);
    return KGE_EINVAL;
  }
  if (p->hidden_size != ACRE_K) {
    set_error("%s: unsupported hidden_size %d (the trunk views each row as 10 x 20: needs 200)", fn, p->hidden_size);
    return KGE_ENOTSUP;
  }
  if (p->way == 0 && acre_tr_serial_smem(C).total * (long long)sizeof(float) > ACRE_SMEM_MAX) {
    set_error("%s: serial in_channels %d exceeds the shared-memory bound (C <= 46)", fn, C);
    return KGE_ENOTSUP;
  }
  if (p->way == 1 && C > ACRE_TR_PAR_MAX) {
    set_error("%s: parallel in_channels %d above %d", fn, C, ACRE_TR_PAR_MAX);
    return KGE_ENOTSUP;
  }
  return KGE_OK;
}

// the 18 parameter pointers in the gradient order of kge_acre_train_bwd
static void acre_train_ptrs(const kge_acre_train_t* p, const float* out[KGE_ACRE_TRAIN_GRADS]) {
  const float* v[KGE_ACRE_TRAIN_GRADS] = {p->ent, p->rel, p->bn0_weight, p->bn0_bias, p->conv1_weight, p->conv1_bias,
                                          p->conv2_weight, p->conv2_bias, p->conv3_weight, p->conv3_bias,
                                          p->W_gate_e_weight, p->W_gate_e_bias, p->bn1_weight, p->bn1_bias,
                                          p->fc_weight, p->fc_bias, p->bn2_weight, p->bn2_bias};
  for (int i = 0; i < KGE_ACRE_TRAIN_GRADS; ++i) out[i] = v[i];
}

// slot i is present for this configuration: conv biases with acre_bias only, W_gate_e in the parallel way only
static bool acre_train_present(const kge_acre_train_t* p, int i) {
  if (i == 5 || i == 7 || i == 9) return p->conv1_bias != nullptr;
  if (i == 10 || i == 11) return p->way == 1;
  return true;
}

// KGE_OK, or the error code of an unsupported geometry / malformed call (message set for `fn`)
static int acre_train_check(const kge_acre_train_t* p, const char* fn, int64_t Q, int64_t B) {
  if (!p) { set_error("%s: null pointer", fn); return KGE_EINVAL; }
  if (int rc = acre_train_shape(p, fn)) return rc;
  const int nbias = (p->conv1_bias != nullptr) + (p->conv2_bias != nullptr) + (p->conv3_bias != nullptr);
  if (nbias != 0 && nbias != 3) {
    set_error("%s: conv biases must be all set (acre_bias) or all NULL", fn);
    return KGE_EINVAL;
  }
  const float* ptrs[KGE_ACRE_TRAIN_GRADS];
  acre_train_ptrs(p, ptrs);
  for (int i = 0; i < KGE_ACRE_TRAIN_GRADS; ++i)
    if (acre_train_present(p, i) && !ptrs[i]) { set_error("%s: null parameter tensor %d", fn, i); return KGE_EINVAL; }
  const float* run[] = {p->bn0_mean, p->bn0_var, p->bn1_mean, p->bn1_var, p->bn2_mean, p->bn2_var};
  int nrun = 0;
  for (const float* t : run) nrun += t != nullptr;
  if (nrun != 0 && nrun != 6) { set_error("%s: running statistics must be all set or all NULL", fn); return KGE_EINVAL; }
  const long long rows = p->way == 1 ? Q * p->in_channels : Q;
  if (B < 2 || Q < B || Q % B != 0 || Q > 0x7fffffffll || (rows + PBM - 1) / PBM > 65535) {
    set_error("%s: bad Q %lld / B %lld (Q a multiple of B >= 2)", fn, (long long)Q, (long long)B);
    return KGE_EINVAL;
  }
  return KGE_OK;
}

static AcreTrain acre_train_args(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                                 const float* noise0, const float* noise1, float* ws) {
  AcreTrain a{};
  a.ent = p->ent; a.rel = p->rel; a.e = e; a.r = r;
  a.C = p->in_channels; a.dil[0] = p->first_atrous; a.dil[1] = p->second_atrous; a.dil[2] = p->third_atrous;
  a.par = p->way == 1; a.has_bias = p->conv1_bias != nullptr; a.Q = Q; a.B = B;
  a.bn0_w = p->bn0_weight; a.bn0_b = p->bn0_bias;
  a.conv_w[0] = p->conv1_weight; a.conv_w[1] = p->conv2_weight; a.conv_w[2] = p->conv3_weight;
  a.conv_b[0] = p->conv1_bias; a.conv_b[1] = p->conv2_bias; a.conv_b[2] = p->conv3_bias;
  a.bn1_w = p->bn1_weight; a.bn1_b = p->bn1_bias; a.noise0 = noise0; a.noise1 = noise1;
  const AcreTrainLayout L = acre_train_layout(Q, B, a.C, a.par);
  a.img = ws + L.img; a.y = ws + L.y; a.feat = ws + L.feat; a.a1 = ws + L.a1; a.a2 = ws + L.a2; a.gate = ws + L.gate;
  a.st0 = ws + L.st0; a.st1 = ws + L.st1; a.part0 = ws + L.part0; a.part1 = ws + L.part1; a.red1 = ws + L.red1;
  a.dimg = ws + L.dimg;
  for (int l = 0; l < 3; ++l) { a.pw[l] = ws + L.pw[l]; a.pb[l] = ws + L.pb[l]; }
  return a;
}

static int acre_tr_smem_optin(const void* kernel, size_t bytes) {
  if (bytes > 48 * 1024) KGE_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return KGE_OK;
}

int64_t kge_acre_train_workspace_bytes(const kge_acre_train_t* p, int64_t Q, int64_t B) {
  if (!p || B < 1 || acre_train_shape(p, "kge_acre_train_workspace_bytes")) return 0;
  return acre_train_layout(Q > B ? Q : B, B, p->in_channels, p->way == 1).total * (int64_t)sizeof(float);
}

int kge_acre_train_fwd(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                       const float* noise0, const float* noise1, const float* noise2, float* x, void* workspace,
                       int64_t workspace_bytes, void* stream) {
  if (int rc = acre_train_check(p, "kge_acre_train_fwd", Q, B)) return rc;
  if (!e || !r || !x || !workspace) { set_error("kge_acre_train_fwd: null pointer"); return KGE_EINVAL; }
  if (workspace_bytes < kge_acre_train_workspace_bytes(p, Q, B)) {
    set_error("kge_acre_train_fwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const AcreTrain a = acre_train_args(p, e, r, Q, B, noise0, noise1, ws);
  const AcreTrainLayout L = acre_train_layout(Q, B, a.C, a.par);
  const ConveTrain cv = acre_tr_view(a, p->bn2_weight, p->bn2_bias, noise2, ws + L.hpre, ws + L.st2, ws + L.red0);
  const int C = a.C;
  const long long Fw = acre_feat_width(C);
  conve_tr_gather_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(cv);
  KGE_CHECK_LAUNCH("conve_tr_gather_kernel<acre>");
  conve_tr_bn_stats_kernel<<<1, 256, 0, st>>>(a.part0, Q, B, 1, (float)ACRE_PIX, p->bn0_eps, p->bn0_momentum, a.st0,
                                              p->bn0_mean, p->bn0_var);
  KGE_CHECK_LAUNCH("conve_tr_bn_stats_kernel<acre bn0>");
  if (!a.par) {
    const size_t smem = (size_t)acre_tr_serial_smem(C).total * sizeof(float);
    if (int rc = acre_tr_smem_optin((const void*)acre_tr_serial_kernel, smem)) return rc;
    acre_tr_serial_kernel<<<(unsigned)Q, ACRE_THREADS, smem, st>>>(a);
    KGE_CHECK_LAUNCH("acre_tr_serial_kernel");
  } else {
    const size_t smem = (size_t)acre_tr_gate_smem(C) * sizeof(float);
    if (int rc = acre_tr_smem_optin((const void*)acre_tr_gate_kernel, smem)) return rc;
    acre_tr_gate_kernel<<<(unsigned)Q, ACRE_GATE_THREADS, smem, st>>>(a);
    KGE_CHECK_LAUNCH("acre_tr_gate_kernel");
    const long long rows = Q * C;
    if (int rc = launch_gemm<EPI_STORE>(acre_plan_gate(a.gate, p->W_gate_e_weight, p->W_gate_e_bias, rows, a.y,
                                                       pick_tile(rows, ACRE_PIX)), st, "proj_gemm_kernel<acre train gate>"))
      return rc;
  }
  acre_tr_bn1_part_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("acre_tr_bn1_part_kernel");
  conve_tr_bn_stats_kernel<<<proj_tiles(C, 256), 256, 0, st>>>(a.part1, Q, B, C, (float)ACRE_PIX, p->bn1_eps,
                                                              p->bn1_momentum, a.st1, p->bn1_mean, p->bn1_var);
  KGE_CHECK_LAUNCH("conve_tr_bn_stats_kernel<acre bn1>");
  acre_tr_feat_kernel<<<proj_tiles(Q * Fw, 256), 256, 0, st>>>(a);
  KGE_CHECK_LAUNCH("acre_tr_feat_kernel");
  float* partial = ws + L.partial;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_fc(a.feat, p->fc_weight, Q, Fw, ACRE_K, partial), st,
                                      "proj_gemm_kernel<acre train fc>")) return rc;
  conve_tr_fc_combine_kernel<<<proj_tiles(Q * ACRE_K, 256), 256, 0, st>>>(partial, conve_fc_slices(Fw), Q * ACRE_K,
                                                                          ACRE_K, p->fc_bias, noise2, cv.hpre);
  KGE_CHECK_LAUNCH("conve_tr_fc_combine_kernel<acre>");
  conve_tr_bn2_kernel<<<proj_tiles(ACRE_K, 256), 256, 0, st>>>(cv, p->bn2_eps, p->bn2_momentum, p->bn2_mean,
                                                               p->bn2_var, x);
  KGE_CHECK_LAUNCH("conve_tr_bn2_kernel<acre>");
  return KGE_OK;
}

int kge_acre_train_bwd(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                       const float* noise0, const float* noise1, const float* noise2, const float* gx, const float* x,
                       float* const* grads, void* workspace, int64_t workspace_bytes, void* stream) {
  if (int rc = acre_train_check(p, "kge_acre_train_bwd", Q, B)) return rc;
  if (!e || !r || !gx || !x || !grads || !workspace) {
    set_error("kge_acre_train_bwd: null pointer");
    return KGE_EINVAL;
  }
  for (int i = 0; i < KGE_ACRE_TRAIN_GRADS; ++i)
    if ((grads[i] != nullptr) != acre_train_present(p, i)) {
      set_error("kge_acre_train_bwd: gradient slot %d must be %s", i, acre_train_present(p, i) ? "set" : "NULL");
      return KGE_EINVAL;
    }
  if (workspace_bytes < kge_acre_train_workspace_bytes(p, Q, B)) {
    set_error("kge_acre_train_bwd: workspace too small");
    return KGE_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = (float*)workspace;
  const AcreTrain a = acre_train_args(p, e, r, Q, B, noise0, noise1, ws);
  const AcreTrainLayout L = acre_train_layout(Q, B, a.C, a.par);
  const ConveTrain cv = acre_tr_view(a, p->bn2_weight, p->bn2_bias, noise2, ws + L.hpre, ws + L.st2, ws + L.red0);
  const int C = a.C;
  const long long Fw = acre_feat_width(C);
  float* dh = ws + L.dh;
  // grads: ent, rel, bn0.w, bn0.b, conv1.w, conv1.b, conv2.w, conv2.b, conv3.w, conv3.b, W_gate_e.w, W_gate_e.b,
  //        bn1.w, bn1.b, fc.w, fc.b, bn2.w, bn2.b
  conve_tr_bn2_bwd_kernel<<<proj_tiles(ACRE_K, 256), 256, 0, st>>>(cv, gx, x, dh, grads[16], grads[17], grads[15]);
  KGE_CHECK_LAUNCH("conve_tr_bn2_bwd_kernel<acre>");
  // d fc.weight reads feat before d feat overwrites it (same stream, in order)
  if (int rc = launch_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(dh, a.feat, Q, Fw, ACRE_K, grads[14]), st,
                                       "proj_gemm_kernel<acre grad fc_w>")) return rc;
  if (int rc = launch_gemm<EPI_STORE>(conve_plan_grad_feat(dh, p->fc_weight, Q, Fw, ACRE_K, a.feat), st,
                                      "proj_gemm_kernel<acre grad feat>")) return rc;
  acre_tr_bn1_bwd_part_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("acre_tr_bn1_bwd_part_kernel");
  conve_tr_reduce_kernel<<<proj_tiles(C, 256), 256, 0, st>>>(a.part1, Q, B, C, a.red1, grads[12], grads[13]);
  KGE_CHECK_LAUNCH("conve_tr_reduce_kernel<acre bn1>");
  acre_tr_bn1_bwd_kernel<<<proj_tiles(Q * Fw, 256), 256, 0, st>>>(a);
  KGE_CHECK_LAUNCH("acre_tr_bn1_bwd_kernel");
  if (!a.par) {
    const size_t smem = (size_t)acre_tr_serial_smem(C).total * sizeof(float);
    if (int rc = acre_tr_smem_optin((const void*)acre_tr_serial_bwd_kernel, smem)) return rc;
    acre_tr_serial_bwd_kernel<<<(unsigned)Q, ACRE_THREADS, smem, st>>>(a);
    KGE_CHECK_LAUNCH("acre_tr_serial_bwd_kernel");
  } else {
    const long long rows = Q * C;
    // d W_gate_e.weight reads the gate rows before d gate overwrites them
    if (int rc = launch_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(a.feat, a.gate, rows, ACRE_GATE, ACRE_PIX, grads[10]),
                                         st, "proj_gemm_kernel<acre grad W_gate_e>")) return rc;
    conve_tr_colsum_kernel<<<proj_tiles(ACRE_PIX, 256), 256, 0, st>>>(a.feat, rows, ACRE_PIX, grads[11]);
    KGE_CHECK_LAUNCH("conve_tr_colsum_kernel<acre W_gate_e.bias>");
    if (int rc = launch_gemm<EPI_STORE>(conve_plan_grad_feat(a.feat, p->W_gate_e_weight, rows, ACRE_GATE, ACRE_PIX,
                                                             a.gate), st, "proj_gemm_kernel<acre grad gate>"))
      return rc;
    const size_t smem = (size_t)acre_tr_gate_bwd_smem(C) * sizeof(float);
    if (int rc = acre_tr_smem_optin((const void*)acre_tr_gate_bwd_kernel, smem)) return rc;
    acre_tr_gate_bwd_kernel<<<(unsigned)Q, ACRE_GATE_THREADS, smem, st>>>(a);
    KGE_CHECK_LAUNCH("acre_tr_gate_bwd_kernel");
  }
  for (int l = 0; l < 3; ++l) {
    const int nw = C * acre_tr_cin(l, C, a.par) * 9;
    conve_tr_colsum_kernel<<<proj_tiles(nw, 256), 256, 0, st>>>(a.pw[l], Q, nw, grads[4 + 2 * l]);
    KGE_CHECK_LAUNCH("conve_tr_colsum_kernel<acre conv weight>");
    if (a.has_bias) {
      conve_tr_colsum_kernel<<<proj_tiles(C, 256), 256, 0, st>>>(a.pb[l], Q, C, grads[5 + 2 * l]);
      KGE_CHECK_LAUNCH("conve_tr_colsum_kernel<acre conv bias>");
    }
  }
  acre_tr_bn0_part_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(a);
  KGE_CHECK_LAUNCH("acre_tr_bn0_part_kernel");
  conve_tr_reduce_kernel<<<1, 256, 0, st>>>(a.part0, Q, B, 1, cv.red0, grads[2], grads[3]);
  KGE_CHECK_LAUNCH("conve_tr_reduce_kernel<acre bn0>");
  conve_tr_bn0_bwd_kernel<<<(unsigned)Q, CONVE_TR_THREADS, 0, st>>>(cv, grads[0], grads[1]);
  KGE_CHECK_LAUNCH("conve_tr_bn0_bwd_kernel<acre>");
  return KGE_OK;
}

}  // extern "C"
