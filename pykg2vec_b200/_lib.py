"""ctypes binding of libkge_b200.so (the C-ABI declared in include/kge_b200.h).

There is no fallback: if the library is missing or a call fails this module raises.
torch is used only for device memory, streams and tensor metadata.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_build", "libkge_b200.so")
MAX_TABLES = 16
ABI_VERSION = 10
ENOTSUP = -2   # include/kge_b200.h KGE_ENOTSUP

MODEL_IDS = {
    "transe": 0, "transh": 1, "transd": 2, "transr": 3, "rotate": 4, "hole": 5,
    "distmult": 6, "complex": 7, "cp": 8, "simple": 9, "transm": 10, "rescal": 11, "analogy": 12,
    "simple_ignr": 13, "quate": 14, "octonione": 15, "kg2e": 16, "slm": 17, "sme": 18, "sme_bl": 19, "ntn": 20, "convkb": 21,
}
GROUP_TAIL, GROUP_HEAD = 0, 1
RANK_FORCE_GATHER, RANK_TAIL_ONLY, RANK_HEAD_ONLY = 1, 2, 4
RANK_SINGLE_STREAM, RANK_NO_TC, RANK_PROFILE = 8, 16, 32

# every symbol include/kge_b200.h declares (tests check they are all exported)
EXPORTS = [
    "kge_abi_version", "kge_version", "kge_last_error", "kge_launch_count",
    "kge_score_fwd", "kge_score_bwd", "kge_normalize_rows",
    "kge_loss_pairwise_hinge", "kge_loss_pointwise_logistic", "kge_loss_selfadv", "kge_reg_fwd_bwd",
    "kge_train_pairwise_hinge_sgd", "kge_train_pointwise_logistic", "kge_train_pairwise_selfadv", "kge_optim_apply_rows", "kge_optim_apply_dense",
    "kge_rank_workspace_bytes", "kge_rank_1vsall", "kge_rank_tc_probe", "kge_rank_last_sweep_ms", "kge_rank_last_sweep_directions", "kge_debug_set_tc_trace",
    "kge_tripleset_capacity", "kge_tripleset_build", "kge_sample_negatives",
    "kge_proj_tail_fwd", "kge_proj_tail_bwd", "kge_proj_bce", "kge_proj_rank_workspace_bytes", "kge_proj_rank", "kge_proj_labels",
    "kge_conve_trunk_workspace_bytes", "kge_conve_trunk_fwd", "kge_hyper_trunk_workspace_bytes", "kge_hyper_trunk_fwd",
    "kge_interacte_trunk_workspace_bytes", "kge_interacte_trunk_fwd",
    "kge_acre_trunk_workspace_bytes", "kge_acre_trunk_fwd",
    "kge_proje_trunk_fwd", "kge_proje_train_step", "kge_reg_l1_dense", "kge_proj_labels_negatives",
    "kge_tucker_workspace_bytes", "kge_tucker_cores", "kge_tucker_trunk_fwd", "kge_tucker_trunk_bwd",
    "kge_tucker_cores_bwd", "kge_tucker_mask1",
    "kge_conve_train_workspace_bytes", "kge_conve_train_fwd", "kge_conve_train_bwd",
    "kge_hyper_train_workspace_bytes", "kge_hyper_train_fwd", "kge_hyper_train_bwd",
    "kge_interacte_train_workspace_bytes", "kge_interacte_train_fwd", "kge_interacte_train_bwd",
    "kge_acre_train_workspace_bytes", "kge_acre_train_fwd", "kge_acre_train_bwd",
    "kge_project_entities", "kge_normalize_rows_to",
]


class KgeModel(ctypes.Structure):
    _fields_ = [
        ("model", ctypes.c_int32), ("dim", ctypes.c_int32), ("rel_dim", ctypes.c_int32),
        ("l1_flag", ctypes.c_int32), ("margin", ctypes.c_float), ("phase_scale", ctypes.c_float),
        ("num_ent", ctypes.c_int64), ("num_rel", ctypes.c_int64),
        ("tables", ctypes.c_void_p * MAX_TABLES),
    ]


class KgeError(RuntimeError):
    pass


class KgeNotSupported(KgeError):
    """KGE_ENOTSUP: the entry point has no kernel for this model / shape (callers with an alternative path
    catch exactly this; every other error propagates)."""


_lib = None


def lib():
    """Load the shared library (once).  Raises if it has not been built: the product
    path never falls back to a CPU or PyTorch implementation."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise KgeError("libkge_b200.so not found at %s — run `python -m pykg2vec_b200.build` "
                       "(or __graft_entry__.build())" % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    L.kge_version.restype = ctypes.c_char_p
    L.kge_last_error.restype = ctypes.c_char_p
    L.kge_launch_count.restype = ctypes.c_int64
    L.kge_rank_workspace_bytes.restype = ctypes.c_int64
    L.kge_tripleset_capacity.restype = ctypes.c_int64
    L.kge_proj_rank_workspace_bytes.restype = ctypes.c_int64
    L.kge_conve_trunk_workspace_bytes.restype = ctypes.c_int64
    L.kge_hyper_trunk_workspace_bytes.restype = ctypes.c_int64
    L.kge_interacte_trunk_workspace_bytes.restype = ctypes.c_int64
    L.kge_acre_trunk_workspace_bytes.restype = ctypes.c_int64
    L.kge_tucker_workspace_bytes.restype = ctypes.c_int64
    L.kge_conve_train_workspace_bytes.restype = ctypes.c_int64
    L.kge_hyper_train_workspace_bytes.restype = ctypes.c_int64
    L.kge_interacte_train_workspace_bytes.restype = ctypes.c_int64
    L.kge_acre_train_workspace_bytes.restype = ctypes.c_int64
    if L.kge_abi_version() != ABI_VERSION:
        raise KgeError("libkge_b200.so ABI %d != binding ABI %d" % (L.kge_abi_version(), ABI_VERSION))
    missing = [name for name in EXPORTS if not hasattr(L, name)]
    if missing:   # a library built before entry points were added to this ABI version: rebuild it
        raise KgeError("libkge_b200.so at %s lacks %s — rebuild it (python -m pykg2vec_b200.build)"
                       % (LIB_PATH, ", ".join(missing)))
    _lib = L
    return L


def check(rc, what):
    if rc != 0:
        raise (KgeNotSupported if rc == ENOTSUP else KgeError)("%s failed (%d): %s" % (what, rc, lib().kge_last_error().decode()))


def _ptr(t):
    if t is None:
        return ctypes.c_void_p(0)
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev_i64(t, name):
    if t.dtype != torch.int64 or not t.is_cuda or not t.is_contiguous():
        raise KgeError("%s must be a contiguous CUDA int64 tensor" % name)
    return t


def _dev_f32(t, name):
    if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
        raise KgeError("%s must be a contiguous CUDA float32 tensor" % name)
    return t


class ModelDesc:
    """Host description of a model: C-ABI name + device tables in C-ABI order."""

    def __init__(self, name, tables, dim, rel_dim=None, l1_flag=False, margin=0.0, phase_scale=0.0,
                 num_ent=None, num_rel=None):
        self.name = name.lower()
        if self.name not in MODEL_IDS:
            raise KgeError("unknown model %r" % name)
        self.tables = [_dev_f32(t, "table") for t in tables]
        self.dim = int(dim)
        self.rel_dim = int(rel_dim if rel_dim is not None else dim)
        self.l1_flag = bool(l1_flag)
        self.margin = float(margin)
        self.phase_scale = float(phase_scale)
        rel_index = {"rotate": 2, "complex": 2, "simple": 2, "simple_ignr": 2, "quate": 4,
                     "octonione": 8, "kg2e": 2}.get(self.name, 1)
        self.num_ent = int(num_ent if num_ent is not None else self.tables[0].shape[0])
        self.num_rel = int(num_rel if num_rel is not None else self.tables[rel_index].shape[0])

    def c_struct(self, tables=None):
        m = KgeModel()
        m.model = MODEL_IDS[self.name]
        m.dim, m.rel_dim, m.l1_flag = self.dim, self.rel_dim, int(self.l1_flag)
        m.margin, m.phase_scale = self.margin, self.phase_scale
        m.num_ent, m.num_rel = self.num_ent, self.num_rel
        for k, t in enumerate(tables if tables is not None else self.tables):
            m.tables[k] = t.data_ptr()
        return m


def _table_ptr_array(tensors):
    arr = (ctypes.c_void_p * MAX_TABLES)()
    for k, t in enumerate(tensors):
        arr[k] = t.data_ptr() if t is not None else None
    return arr


def score_fwd(desc, h, r, t, grouping=GROUP_TAIL, out=None):
    h, r, t = _dev_i64(h, "h"), _dev_i64(r, "r"), _dev_i64(t, "t")
    n = h.numel()
    if r.numel() != n or t.numel() != n:
        raise KgeError("h, r, t must have equal length")
    if out is None:
        out = torch.empty(n, dtype=torch.float32, device=h.device)
    m = desc.c_struct()
    check(lib().kge_score_fwd(ctypes.byref(m), int(grouping), _ptr(h), _ptr(r), _ptr(t),
                              ctypes.c_int64(n), _ptr(out), _stream()), "kge_score_fwd")
    return out


def score_bwd(desc, h, r, t, grad_scores, grad_tables):
    m = desc.c_struct()
    arr = _table_ptr_array(grad_tables)
    check(lib().kge_score_bwd(ctypes.byref(m), _ptr(h), _ptr(r), _ptr(t), ctypes.c_int64(h.numel()),
                              _ptr(_dev_f32(grad_scores, "grad_scores")), arr, _stream()), "kge_score_bwd")


def normalize_rows(table):
    """Rescal.get_normalized_data (pairwise.py:862-865): rows / ||row||_2, IN PLACE."""
    t = _dev_f32(table, "table")
    check(lib().kge_normalize_rows(_ptr(t), ctypes.c_int64(t.shape[0]), ctypes.c_int64(t.shape[1]), _stream()),
          "kge_normalize_rows")
    return table


def loss_pairwise_hinge(pos, neg, margin, want_grad=True):
    pos, neg = _dev_f32(pos, "pos"), _dev_f32(neg, "neg")
    loss = torch.empty(1, dtype=torch.float32, device=pos.device)
    gp = torch.empty_like(pos) if want_grad else None
    gn = torch.empty_like(neg) if want_grad else None
    check(lib().kge_loss_pairwise_hinge(_ptr(pos), _ptr(neg), ctypes.c_int64(pos.numel()),
                                        ctypes.c_float(margin), _ptr(loss), _ptr(gp), _ptr(gn), _stream()),
          "kge_loss_pairwise_hinge")
    return loss, gp, gn


def loss_pointwise_logistic(preds, target, want_grad=True):
    preds, target = _dev_f32(preds, "preds"), _dev_f32(target, "target")
    loss = torch.empty(1, dtype=torch.float32, device=preds.device)
    g = torch.empty_like(preds) if want_grad else None
    check(lib().kge_loss_pointwise_logistic(_ptr(preds), _ptr(target), ctypes.c_int64(preds.numel()),
                                            _ptr(loss), _ptr(g), _stream()), "kge_loss_pointwise_logistic")
    return loss, g


def loss_selfadv(pos, neg, neg_rate, alpha, want_grad=True):
    pos, neg = _dev_f32(pos, "pos"), _dev_f32(neg, "neg")
    if neg.numel() != pos.numel() * neg_rate:
        raise KgeError("neg must hold neg_rate scores per positive")
    loss = torch.empty(1, dtype=torch.float32, device=pos.device)
    gp = torch.empty_like(pos) if want_grad else None
    gn = torch.empty_like(neg) if want_grad else None
    check(lib().kge_loss_selfadv(_ptr(pos), _ptr(neg), ctypes.c_int64(pos.numel()), ctypes.c_int32(neg_rate),
                                 ctypes.c_float(alpha), _ptr(loss), _ptr(gp), _ptr(gn), _stream()),
          "kge_loss_selfadv")
    return loss, gp, gn


def reg_fwd_bwd(desc, reg_type, lmbda, h, r, t, grad_scale=0.0, grad_tables=None):
    out = torch.empty(1, dtype=torch.float32, device=h.device)
    m = desc.c_struct()
    arr = _table_ptr_array(grad_tables) if grad_tables is not None else None
    check(lib().kge_reg_fwd_bwd(ctypes.byref(m), int(reg_type), ctypes.c_float(lmbda), _ptr(h), _ptr(r),
                                _ptr(t), ctypes.c_int64(h.numel()), _ptr(out), ctypes.c_float(grad_scale),
                                arr, _stream()), "kge_reg_fwd_bwd")
    return out


def train_pairwise_hinge_sgd(desc, grad_scratch, ph, pr, pt, nh, nr, nt, margin, lr, loss_out=None):
    """In-place fused step on desc.tables; grad_scratch: zero-filled dense buffers shaped
    like the tables (left zero-filled on return)."""
    if loss_out is None:
        loss_out = torch.empty(1, dtype=torch.float32, device=ph.device)
    m = desc.c_struct()
    rw = _table_ptr_array(desc.tables)
    gs = _table_ptr_array(grad_scratch)
    check(lib().kge_train_pairwise_hinge_sgd(ctypes.byref(m), rw, gs, _ptr(ph), _ptr(pr), _ptr(pt), _ptr(nh),
                                             _ptr(nr), _ptr(nt), ctypes.c_int64(ph.numel()),
                                             ctypes.c_float(margin), ctypes.c_float(lr), _ptr(loss_out),
                                             _stream()), "kge_train_pairwise_hinge_sgd")
    return loss_out


def train_pointwise_logistic(desc, grad_scratch, h, r, t, y, loss_out=None):
    """forward + Criterion.pointwise_logistic + backward of a pointwise batch in one kernel: returns the loss
    [1]; row gradients are accumulated into grad_scratch (dense buffers shaped like the tables)."""
    if loss_out is None:
        loss_out = torch.empty(1, dtype=torch.float32, device=h.device)
    m = desc.c_struct()
    gs = _table_ptr_array(grad_scratch)
    check(lib().kge_train_pointwise_logistic(ctypes.byref(m), gs, _ptr(_dev_i64(h, "h")), _ptr(_dev_i64(r, "r")),
                                             _ptr(_dev_i64(t, "t")), _ptr(_dev_i64(y, "y")), ctypes.c_int64(h.numel()),
                                             _ptr(loss_out), _stream()), "kge_train_pointwise_logistic")
    return loss_out


def train_pairwise_selfadv(desc, grad_scratch, ph, pr, pt, nh, nr, nt, neg_rate, alpha, loss_out=None):
    """RotatE: forward of the positives and their negatives + the self-adversarial loss + backward in one kernel:
    returns the loss [1]; row gradients are accumulated into grad_scratch.  KgeError (KGE_ENOTSUP) when neg_rate
    does not fit a CTA's shared memory — the caller then takes the unfused path."""
    if loss_out is None:
        loss_out = torch.empty(1, dtype=torch.float32, device=ph.device)
    if nh.numel() != ph.numel() * int(neg_rate):
        raise KgeError("self-adversarial loss: %d negatives for %d positives x neg_rate %d"
                       % (nh.numel(), ph.numel(), int(neg_rate)))
    m = desc.c_struct()
    gs = _table_ptr_array(grad_scratch)
    check(lib().kge_train_pairwise_selfadv(
        ctypes.byref(m), gs, _ptr(_dev_i64(ph, "ph")), _ptr(_dev_i64(pr, "pr")), _ptr(_dev_i64(pt, "pt")),
        _ptr(_dev_i64(nh, "nh")), _ptr(_dev_i64(nr, "nr")), _ptr(_dev_i64(nt, "nt")), ctypes.c_int64(ph.numel()),
        ctypes.c_int32(int(neg_rate)), ctypes.c_float(float(alpha)), _ptr(loss_out), _stream()),
        "kge_train_pairwise_selfadv")
    return loss_out


def optim_apply_rows(desc, grad_scratch, state, optimizer, h, r, t, lr, eps=1e-10):
    """optimizer: 0 SGD, 1 Adagrad.  Consumes (and re-zeroes) grad_scratch for the touched rows."""
    m = desc.c_struct()
    rw = _table_ptr_array(desc.tables)
    gs = _table_ptr_array(grad_scratch)
    stt = _table_ptr_array(state) if state is not None else None
    check(lib().kge_optim_apply_rows(ctypes.byref(m), rw, gs, stt, ctypes.c_int(optimizer), _ptr(h), _ptr(r),
                                     _ptr(t), ctypes.c_int64(h.numel()), ctypes.c_float(lr),
                                     ctypes.c_float(eps), _stream()), "kge_optim_apply_rows")


OPT_SGD, OPT_ADAGRAD, OPT_ADAM = 0, 1, 2


def optim_apply_dense(w, grad, optimizer, lr, state1=None, state2=None, eps=None, betas=(0.9, 0.999), step=1):
    """Dense optimizer step on ONE parameter tensor; consumes (and re-zeroes) its dense gradient buffer.
    optimizer: OPT_SGD / OPT_ADAGRAD (state1) / OPT_ADAM (state1 = exp_avg, state2 = exp_avg_sq, step >= 1)."""
    if eps is None:
        eps = 1e-8 if optimizer == OPT_ADAM else 1e-10
    w, grad = _dev_f32(w, "w"), _dev_f32(grad, "grad")
    if grad.numel() != w.numel():
        raise KgeError("gradient buffer must be shaped like the parameter")
    check(lib().kge_optim_apply_dense(_ptr(w), _ptr(grad), _ptr(state1), _ptr(state2), ctypes.c_int64(w.numel()),
                                      ctypes.c_int(optimizer), ctypes.c_float(lr), ctypes.c_float(eps),
                                      ctypes.c_float(betas[0]), ctypes.c_float(betas[1]), ctypes.c_int64(step),
                                      _stream()), "kge_optim_apply_dense")


def rank_workspace_bytes(desc, Q):
    m = desc.c_struct()
    return int(lib().kge_rank_workspace_bytes(ctypes.byref(m), ctypes.c_int64(Q)))


def rank_1vsall(desc, qh, qr, qt, filt_t=None, filt_h=None, counts=None, row_lo=0, row_hi=None,
                query_desc=None, tgt_h=None, tgt_t=None, flags=0, workspace=None):
    """Accumulate 0-based (tail raw, tail filtered, head raw, head filtered) rank counts of the
    queries over candidate rows [row_lo, row_hi) into counts [Q,4] int32.
    filt_* = (ptr[Q+1] int64 cuda, idx[nnz] int64 cuda) or None."""
    qh, qr, qt = _dev_i64(qh, "qh"), _dev_i64(qr, "qr"), _dev_i64(qt, "qt")
    Q = qh.numel()
    if row_hi is None:
        row_hi = row_lo + desc.num_ent
    if counts is None:
        counts = torch.zeros((Q, 4), dtype=torch.int32, device=qh.device)
    nbytes = rank_workspace_bytes(desc, Q)
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=qh.device)
    m = desc.c_struct()
    mq = query_desc.c_struct() if query_desc is not None else None
    ft_ptr, ft_idx = filt_t if filt_t is not None else (None, None)
    fh_ptr, fh_idx = filt_h if filt_h is not None else (None, None)
    check(lib().kge_rank_1vsall(
        ctypes.byref(m), ctypes.byref(mq) if mq is not None else None,
        ctypes.c_int64(row_lo), ctypes.c_int64(row_hi), _ptr(qh), _ptr(qr), _ptr(qt),
        _ptr(tgt_h), _ptr(tgt_t), ctypes.c_int64(Q),
        _ptr(ft_ptr), _ptr(ft_idx), ctypes.c_int64(ft_idx.numel() if ft_idx is not None else 0),
        _ptr(fh_ptr), _ptr(fh_idx), ctypes.c_int64(fh_idx.numel() if fh_idx is not None else 0),
        _ptr(counts), _ptr(workspace), ctypes.c_int64(workspace.numel()), ctypes.c_int(flags), _stream()),
        "kge_rank_1vsall")
    return counts


def rank_last_sweep_directions():
    """how many directions the launch timed by rank_last_sweep_ms(0) swept (2: the tensor-core sweep of a full
    rank call covers tail and head in one launch; 0: nothing profiled)."""
    return int(lib().kge_rank_last_sweep_directions())


def rank_last_sweep_ms(direction):
    """device time (ms) of the main sweep kernel of `direction` in the last rank_1vsall(flags |= RANK_PROFILE)."""
    ms = ctypes.c_float(0.0)
    check(lib().kge_rank_last_sweep_ms(ctypes.c_int(direction), ctypes.byref(ms)), "kge_rank_last_sweep_ms")
    return float(ms.value)


def rank_tc_probe(desc, qh, qr, qt, direction, want_dots=True, query_desc=None, row_lo=0, row_hi=None):
    """Level 1 (tensor cores) of the two-level exact sweep for ONE direction (include/kge_b200.h):
    -> (dots [Q, nc] raw accumulators or None, band, counts [Q,4]); band = (coef [Q,4] = centre, a, b, e per
    query, cn [nc] = norm bound per candidate): the pair (q, c) is certainly better when
    dots - centre > a + b cn + e cn^2, certainly not when dots - centre < -(a + b cn + e cn^2)."""
    qh, qr, qt = _dev_i64(qh, "qh"), _dev_i64(qr, "qr"), _dev_i64(qt, "qt")
    Q = qh.numel()
    if row_hi is None:
        row_hi = row_lo + desc.num_ent
    nc = row_hi - row_lo
    dots = torch.empty((Q, nc), dtype=torch.float32, device=qh.device) if want_dots else None
    tau = torch.empty(Q * 4 + nc, dtype=torch.float32, device=qh.device)
    counts = torch.zeros((Q, 4), dtype=torch.int32, device=qh.device)
    ws = torch.empty(max(rank_workspace_bytes(desc, Q), 16), dtype=torch.uint8, device=qh.device)
    m = desc.c_struct()
    mq = query_desc.c_struct() if query_desc is not None else None
    check(lib().kge_rank_tc_probe(
        ctypes.byref(m), ctypes.byref(mq) if mq is not None else None, ctypes.c_int64(row_lo), ctypes.c_int64(row_hi),
        _ptr(qh), _ptr(qr), _ptr(qt), ctypes.c_int64(Q), ctypes.c_int(direction), _ptr(dots), _ptr(tau),
        _ptr(counts), _ptr(ws), ctypes.c_int64(ws.numel()), _stream()), "kge_rank_tc_probe")
    return dots, (tau[:Q * 4].view(Q, 4), tau[Q * 4:]), counts


def project_entities(desc, r, out=None):
    """TransH / TransD: the projected row of every entity for relation r, [num_ent, dim]
    (include/kge_b200.h kge_project_entities) — TransE over [out, rel] then equals the model."""
    if out is None:
        width = desc.rel_dim if desc.name == "transr" else desc.dim
        out = torch.empty((desc.num_ent, width), dtype=torch.float32, device=desc.tables[0].device)
    m = desc.c_struct()
    check(lib().kge_project_entities(ctypes.byref(m), ctypes.c_int64(int(r)), _ptr(_dev_f32(out, "out")), _stream()),
          "kge_project_entities")
    return out


def normalize_rows_to(table, out=None):
    """F.normalize(table, dim=-1) in the canonical arithmetic into a new tensor (TransR's first
    normalisation of the relation rows, pairwise.py:430-432)."""
    t = _dev_f32(table, "table")
    if out is None:
        out = torch.empty_like(t)
    check(lib().kge_normalize_rows_to(_ptr(t), ctypes.c_int64(t.shape[0]), ctypes.c_int64(t.shape[1]),
                                      _ptr(_dev_f32(out, "out")), _stream()), "kge_normalize_rows_to")
    return out


def tripleset_build(h, r, t, num_ent, num_rel):
    """Hash set of the positive triples on the device -> uint64-as-int64 tensor [capacity]."""
    n = h.numel()
    cap = int(lib().kge_tripleset_capacity(ctypes.c_int64(n)))
    slots = torch.empty(cap, dtype=torch.int64, device=h.device)
    check(lib().kge_tripleset_build(_ptr(_dev_i64(h, "h")), _ptr(_dev_i64(r, "r")), _ptr(_dev_i64(t, "t")),
                                    ctypes.c_int64(n), _ptr(slots), ctypes.c_int64(cap), ctypes.c_int64(num_ent),
                                    ctypes.c_int64(num_rel), _stream()), "kge_tripleset_build")
    return slots


def sample_negatives(slots, ph, pr, pt, neg_rate, head_prob, num_ent, seed, step, layout=0, out=None):
    """layout 0 -> (nh, nr, nt) each [B*neg_rate]; layout 1 -> (h, r, t, y) each [B*(1+neg_rate)]."""
    B = ph.numel()
    n = B * neg_rate if layout == 0 else B * (1 + neg_rate)
    if out is None:
        out = torch.empty((4, n), dtype=torch.int64, device=ph.device)
    check(lib().kge_sample_negatives(_ptr(slots), ctypes.c_int64(slots.numel()), _ptr(_dev_i64(ph, "ph")),
                                     _ptr(_dev_i64(pr, "pr")), _ptr(_dev_i64(pt, "pt")), ctypes.c_int64(B),
                                     ctypes.c_int32(neg_rate), _ptr(head_prob), ctypes.c_int64(num_ent),
                                     ctypes.c_uint64(seed), ctypes.c_uint64(step), ctypes.c_int32(layout),
                                     _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), _ptr(out[3]), _stream()),
          "kge_sample_negatives")
    return (out[0], out[1], out[2]) if layout == 0 else (out[0], out[1], out[2], out[3])


# ---- projection-model tail (include/kge_b200.h: kge_proj_*) ------------------------------------
def _bias_row(bias, N):
    if bias is None:
        return None
    b = _dev_f32(bias, "bias")
    if b.numel() != N:
        raise KgeError("bias must hold one value per entity (%d), got %d" % (N, b.numel()))
    return b


def proj_tail_fwd(x, ent, bias=None, out=None):
    """preds [B,N] = sigmoid(x . ent^T + bias)   (projection.py:100-102)."""
    x, ent = _dev_f32(x, "x"), _dev_f32(ent, "ent")
    if x.dim() != 2 or ent.dim() != 2 or x.shape[1] != ent.shape[1]:
        raise KgeError("x must be [B,k] and ent [N,k]")
    B, k = x.shape
    N = ent.shape[0]
    bias = _bias_row(bias, N)
    if out is None:
        out = torch.empty((B, N), dtype=torch.float32, device=x.device)
    check(lib().kge_proj_tail_fwd(_ptr(x), _ptr(ent), _ptr(bias), ctypes.c_int64(B), ctypes.c_int64(N),
                                  ctypes.c_int32(k), _ptr(out), _stream()), "kge_proj_tail_fwd")
    return out


def proj_tail_bwd(grad_preds, preds, x, ent, grad_x=None, grad_ent=None, grad_bias=None):
    """Accumulates into the given (zero-filled or partially filled) gradient buffers."""
    B, k = x.shape
    N = ent.shape[0]
    check(lib().kge_proj_tail_bwd(_ptr(_dev_f32(grad_preds, "grad_preds")), _ptr(_dev_f32(preds, "preds")),
                                  _ptr(_dev_f32(x, "x")), _ptr(_dev_f32(ent, "ent")), ctypes.c_int64(B),
                                  ctypes.c_int64(N), ctypes.c_int32(k), _ptr(grad_x), _ptr(grad_ent),
                                  _ptr(grad_bias), _stream()), "kge_proj_tail_bwd")


def proj_bce(preds, labels, label_scale=1.0, label_shift=0.0, grad_scale=1.0, want_grad=True):
    """One direction of Criterion.multi_class_bce -> (loss [1], grad_preds [B,N] or None)."""
    preds, labels = _dev_f32(preds, "preds"), _dev_f32(labels, "labels")
    if preds.dim() != 2 or preds.shape != labels.shape:
        raise KgeError("preds and labels must both be [B,N]")
    B, N = preds.shape
    loss = torch.empty(1, dtype=torch.float32, device=preds.device)
    g = torch.empty_like(preds) if want_grad else None
    check(lib().kge_proj_bce(_ptr(preds), _ptr(labels), ctypes.c_int64(B), ctypes.c_int64(N),
                             ctypes.c_float(label_scale), ctypes.c_float(label_shift), ctypes.c_float(grad_scale),
                             _ptr(loss), _ptr(g), _stream()), "kge_proj_bce")
    return loss, g


def proj_labels(rows, ptr, idx, B, N, out=None):
    """Dense [B,N] fp32 label rows (1.0 at the known positives) from a device CSR; rows = CSR row of
    each batch element (None: row b)."""
    ptr, idx = _dev_i64(ptr, "ptr"), _dev_i64(idx, "idx")
    if rows is not None and _dev_i64(rows, "rows").numel() != B:
        raise KgeError("rows must hold one CSR row id per batch element")
    if out is None:
        out = torch.empty((B, N), dtype=torch.float32, device=ptr.device)
    check(lib().kge_proj_labels(_ptr(rows), _ptr(ptr), _ptr(idx), ctypes.c_int64(B), ctypes.c_int64(N),
                                _ptr(_dev_f32(out, "labels")), _stream()), "kge_proj_labels")
    return out


def proj_rank(x, ent, bias, tgt, filt=None, direction=0, counts=None, workspace=None):
    """counts [Q,4] int32 += rank counts of direction 0 (tail: columns 0,1) or 1 (head: 2,3)."""
    x, ent, tgt = _dev_f32(x, "x"), _dev_f32(ent, "ent"), _dev_i64(tgt, "tgt")
    Q, k = x.shape
    N = ent.shape[0]
    bias = _bias_row(bias, N)
    if tgt.numel() != Q:
        raise KgeError("one target id per query row")
    if counts is None:
        counts = torch.zeros((Q, 4), dtype=torch.int32, device=x.device)
    nbytes = int(lib().kge_proj_rank_workspace_bytes(ctypes.c_int64(Q)))
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=x.device)
    fp, fi = filt if filt is not None else (None, None)
    check(lib().kge_proj_rank(_ptr(x), _ptr(ent), _ptr(bias), ctypes.c_int64(Q), ctypes.c_int64(N),
                              ctypes.c_int32(k), _ptr(tgt), _ptr(fp), _ptr(fi),
                              ctypes.c_int64(fi.numel() if fi is not None else 0), ctypes.c_int32(direction),
                              _ptr(counts), _ptr(workspace), ctypes.c_int64(workspace.numel()), _stream()),
          "kge_proj_rank")
    return counts


class KgeConve(ctypes.Structure):
    """kge_conve_t of include/kge_b200.h."""
    _fields_ = [("hidden_size", ctypes.c_int32), ("hidden_size_1", ctypes.c_int32),
                ("bn0_eps", ctypes.c_float), ("bn1_eps", ctypes.c_float)] + \
               [(n, ctypes.c_void_p) for n in ("ent", "rel", "bn0_weight", "bn0_bias", "bn0_mean", "bn0_var",
                                               "conv_weight", "conv_bias", "bn1_weight", "bn1_bias", "bn1_mean",
                                               "bn1_var", "fc_weight", "fc_bias")]


def conve_trunk_fwd(model, e, r, out=None):
    """ConvE inference trunk (projection.py:104-112, :86-99, eval mode): x [Q,k] for entity ids e and
    relation ids r (already offset by tot_relation for the head direction).  `model` is a ConvE with
    the reference's sub-module names."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    if r.numel() != Q:
        raise KgeError("e and r must have equal length")
    tensors = {"ent": model.ent_embeddings.weight, "rel": model.rel_embeddings.weight,
               "bn0_weight": model.bn0.weight, "bn0_bias": model.bn0.bias,
               "bn0_mean": model.bn0.running_mean, "bn0_var": model.bn0.running_var,
               "conv_weight": model.conv2d_1.weight, "conv_bias": model.conv2d_1.bias,
               "bn1_weight": model.bn1.weight, "bn1_bias": model.bn1.bias,
               "bn1_mean": model.bn1.running_mean, "bn1_var": model.bn1.running_var,
               "fc_weight": model.fc.weight, "fc_bias": model.fc.bias}
    p = KgeConve()
    p.hidden_size, p.hidden_size_1 = int(model.hidden_size), int(model.hidden_size_1)
    p.bn0_eps, p.bn1_eps = float(model.bn0.eps), float(model.bn1.eps)
    for name, t in tensors.items():
        setattr(p, name, _dev_f32(t.detach(), name).data_ptr())
    nbytes = int(lib().kge_conve_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q)))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=e.device)
    if out is None:
        out = torch.empty((Q, p.hidden_size), dtype=torch.float32, device=e.device)
    check(lib().kge_conve_trunk_fwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), _ptr(out), _ptr(ws),
                                    ctypes.c_int64(ws.numel()), _stream()), "kge_conve_trunk_fwd")
    return out


HYPER_FIELDS = ("ent", "rel", "bn0_weight", "bn0_bias", "bn0_mean", "bn0_var", "fc1_weight", "fc1_bias",
                "bn1_weight", "bn1_bias", "bn1_mean", "bn1_var", "fc_weight", "fc_bias",
                "bn2_weight", "bn2_bias", "bn2_mean", "bn2_var")


class KgeHyper(ctypes.Structure):
    """kge_hyper_t of include/kge_b200.h."""
    _fields_ = [("ent_hidden_size", ctypes.c_int32), ("rel_hidden_size", ctypes.c_int32), ("num_rel", ctypes.c_int64),
                ("bn0_eps", ctypes.c_float), ("bn1_eps", ctypes.c_float), ("bn2_eps", ctypes.c_float)] + \
               [(n, ctypes.c_void_p) for n in HYPER_FIELDS]


def hyper_trunk_workspace_bytes(ent_hidden_size, rel_hidden_size, num_rel, Q):
    """bytes of device workspace kge_hyper_trunk_fwd needs for Q queries (0 for an unsupported shape)"""
    p = KgeHyper()
    p.ent_hidden_size, p.rel_hidden_size, p.num_rel = int(ent_hidden_size), int(rel_hidden_size), int(num_rel)
    return int(lib().kge_hyper_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q)))


def hyper_trunk_fwd(model, e, r, out=None, workspace=None):
    """HypER inference trunk (projection.py:581-606, eval mode): x [Q,de] for entity ids e and relation ids r
    (both directions pass their own (entity, relation) pair: HypER has no reciprocal relations).  `model` is a
    HypER with the reference's sub-module names.  `workspace`: optional uint8 device buffer, grown if too small."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    if r.numel() != Q:
        raise KgeError("e and r must have equal length")
    mods = {"bn0": model.bn0, "bn1": model.bn1, "bn2": model.bn2}
    tensors = {"ent": model.ent_embeddings.weight, "rel": model.rel_embeddings.weight,
               "fc1_weight": model.fc1.weight, "fc1_bias": model.fc1.bias,
               "fc_weight": model.fc.weight, "fc_bias": model.fc.bias}
    for name, bn in mods.items():
        tensors.update({name + "_weight": bn.weight, name + "_bias": bn.bias,
                        name + "_mean": bn.running_mean, name + "_var": bn.running_var})
    p = KgeHyper()
    p.ent_hidden_size, p.rel_hidden_size = int(model.ent_hidden_size), int(model.rel_hidden_size)
    p.num_rel = int(model.rel_embeddings.weight.shape[0])
    p.bn0_eps, p.bn1_eps, p.bn2_eps = float(model.bn0.eps), float(model.bn1.eps), float(model.bn2.eps)
    for name in HYPER_FIELDS:
        setattr(p, name, _dev_f32(tensors[name].detach(), name).data_ptr())
    nbytes = int(lib().kge_hyper_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q)))
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=e.device)
    if out is None:
        out = torch.empty((Q, p.ent_hidden_size), dtype=torch.float32, device=e.device)
    check(lib().kge_hyper_trunk_fwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), _ptr(out), _ptr(workspace),
                                    ctypes.c_int64(workspace.numel()), _stream()), "kge_hyper_trunk_fwd")
    return out


INTERACTE_FIELDS = ("ent", "rel", "bn0_weight", "bn0_bias", "bn0_mean", "bn0_var", "conv_filt",
                    "bn1_weight", "bn1_bias", "bn1_mean", "bn1_var", "fc_weight", "fc_bias",
                    "bn2_weight", "bn2_bias", "bn2_mean", "bn2_var")
# upper bound of the workspace one kge_interacte_trunk_fwd call may use: the features alone take 150 KB per
# query at the default shape (1, 96, 9, 20x10), 400 KB at (4, 64, 7, 20x10), so a large batch is split into
# chunks of queries (independent of each other: the result is the same bits as one call)
INTERACTE_WORKSPACE_CAP = 256 << 20


class KgeInteracte(ctypes.Structure):
    """kge_interacte_t of include/kge_b200.h."""
    _fields_ = [("feature_permutation", ctypes.c_int32), ("num_filters", ctypes.c_int32),
                ("kernel_size", ctypes.c_int32), ("reshape_height", ctypes.c_int32),
                ("reshape_width", ctypes.c_int32), ("num_rel", ctypes.c_int64),
                ("bn0_eps", ctypes.c_float), ("bn1_eps", ctypes.c_float), ("bn2_eps", ctypes.c_float),
                ("perm", ctypes.c_void_p)] + [(n, ctypes.c_void_p) for n in INTERACTE_FIELDS]


def interacte_struct(P, F, ks, reshape_height, reshape_width, num_rel):
    """a KgeInteracte holding the geometry only (pointers NULL)"""
    p = KgeInteracte()
    p.feature_permutation, p.num_filters, p.kernel_size = int(P), int(F), int(ks)
    p.reshape_height, p.reshape_width, p.num_rel = int(reshape_height), int(reshape_width), int(num_rel)
    return p


def interacte_trunk_workspace_bytes(P, F, ks, reshape_height, reshape_width, num_rel, Q):
    """bytes of device workspace ONE kge_interacte_trunk_fwd call needs for Q queries (0 for an unsupported
    shape)"""
    p = interacte_struct(P, F, ks, reshape_height, reshape_width, num_rel)
    return int(lib().kge_interacte_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q)))


def interacte_trunk_fwd(model, e, r, out=None, workspace=None, cap=None, perm=None):
    """InteractE inference trunk (projection.py:425-442, eval mode): x [Q,k] for entity ids e and relation ids r
    (both directions pass their own (entity, relation) pair: InteractE has no reciprocal relations).  `model` is
    an InteractE with the reference's sub-module names; its chequer permutation is model.chequer_perm.  The
    queries run in chunks whose workspace stays under `cap` bytes (default INTERACTE_WORKSPACE_CAP; a single
    query always runs).  `workspace`: optional uint8 device buffer, grown if too small.  `perm`: the chequer
    permutation already on e's device (default: model.chequer_perm, copied there if needed)."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    if r.numel() != Q:
        raise KgeError("e and r must have equal length")
    mods = {"bn0": model.bn0, "bn1": model.bn1, "bn2": model.bn2}
    tensors = {"ent": model.ent_embeddings.weight, "rel": model.rel_embeddings.weight, "conv_filt": model.conv_filt,
               "fc_weight": model.fc.weight, "fc_bias": model.fc.bias}
    for name, bn in mods.items():
        tensors.update({name + "_weight": bn.weight, name + "_bias": bn.bias,
                        name + "_mean": bn.running_mean, name + "_var": bn.running_var})
    p = interacte_struct(model.feature_permutation, model.num_filters, model.kernel_size, model.reshape_height,
                         model.reshape_width, model.rel_embeddings.weight.shape[0])
    p.bn0_eps, p.bn1_eps, p.bn2_eps = float(model.bn0.eps), float(model.bn1.eps), float(model.bn2.eps)
    for name in INTERACTE_FIELDS:
        setattr(p, name, _dev_f32(tensors[name].detach(), name).data_ptr())
    perm = model.chequer_perm if perm is None else perm
    if perm.device != e.device or perm.dtype != torch.int64:
        perm = perm.to(device=e.device, dtype=torch.int64)
    p.perm = _dev_i64(perm.contiguous(), "chequer_perm").data_ptr()
    k = int(model.reshape_width) * int(model.reshape_height)
    if out is None:
        out = torch.empty((Q, k), dtype=torch.float32, device=e.device)
    per_query = int(lib().kge_interacte_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(1)))
    if per_query == 0:    # unsupported shape: the call below reports why
        chunk = max(Q, 1)
    else:
        chunk = max(1, min(max(Q, 1), int(INTERACTE_WORKSPACE_CAP if cap is None else cap) // per_query))
    nbytes = int(lib().kge_interacte_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(chunk)))
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=e.device)
    for q0 in range(0, max(Q, 1), chunk):
        n = min(chunk, Q - q0)
        check(lib().kge_interacte_trunk_fwd(ctypes.byref(p), _ptr(e[q0:q0 + n]), _ptr(r[q0:q0 + n]),
                                            ctypes.c_int64(n), _ptr(out[q0:q0 + n]), _ptr(workspace),
                                            ctypes.c_int64(workspace.numel()), _stream()), "kge_interacte_trunk_fwd")
    return out


ACRE_FIELDS = ("ent", "rel", "bn0_weight", "bn0_bias", "bn0_mean", "bn0_var", "conv1_weight", "conv1_bias",
               "conv2_weight", "conv2_bias", "conv3_weight", "conv3_bias", "W_gate_e_weight", "W_gate_e_bias",
               "bn1_weight", "bn1_bias", "bn1_mean", "bn1_var", "fc_weight", "fc_bias",
               "bn2_weight", "bn2_bias", "bn2_mean", "bn2_var")
ACRE_WAYS = {"serial": 0, "parallel": 1}
# upper bound of the workspace one kge_acre_trunk_fwd call may use: per query the features take 51 KB at
# in_channels 32 (serial) and the parallel way's W_gate_e input another 205 KB, so an Evaluator-sized batch is
# split into chunks of queries (independent of each other: the result is the same bits as one call)
ACRE_WORKSPACE_CAP = 256 << 20


class KgeAcre(ctypes.Structure):
    """kge_acre_t of include/kge_b200.h."""
    _fields_ = [("in_channels", ctypes.c_int32), ("way", ctypes.c_int32), ("first_atrous", ctypes.c_int32),
                ("second_atrous", ctypes.c_int32), ("third_atrous", ctypes.c_int32), ("hidden_size", ctypes.c_int32),
                ("num_rel", ctypes.c_int64),
                ("bn0_eps", ctypes.c_float), ("bn1_eps", ctypes.c_float), ("bn2_eps", ctypes.c_float)] + \
        [(n, ctypes.c_void_p) for n in ACRE_FIELDS]


def acre_struct(way, in_channels, atrous, hidden_size, num_rel):
    """a KgeAcre holding the configuration only (pointers NULL).  way: "serial" / "parallel" (or 0 / 1; any other
    value is passed on as -1 so that the call reports it); atrous: the three rates."""
    p = KgeAcre()
    p.way = ACRE_WAYS.get(way, way if way in (0, 1) else -1)
    p.in_channels, p.hidden_size, p.num_rel = int(in_channels), int(hidden_size), int(num_rel)
    p.first_atrous, p.second_atrous, p.third_atrous = (int(a) for a in atrous)
    return p


def acre_trunk_workspace_bytes(way, in_channels, atrous, hidden_size, num_rel, Q):
    """bytes of device workspace ONE kge_acre_trunk_fwd call needs for Q queries (0 for an unsupported or
    malformed configuration)"""
    p = acre_struct(way, in_channels, atrous, hidden_size, num_rel)
    return int(lib().kge_acre_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q)))


def acre_trunk_fwd(model, e, r, out=None, workspace=None, cap=None):
    """AcrE inference trunk (projection.py:706-734, eval mode): x [Q,200] for entity ids e and relation ids r
    (both directions pass their own (entity, relation) pair: AcrE indexes rel_embeddings with r as given).
    `model` is an AcrE with the reference's sub-module names.  The queries run in chunks whose workspace stays
    under `cap` bytes (default ACRE_WORKSPACE_CAP; a single query always runs).  `workspace`: optional uint8
    device buffer, grown if too small."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    if r.numel() != Q:
        raise KgeError("e and r must have equal length")
    tensors = {"ent": model.ent_embeddings.weight, "rel": model.rel_embeddings.weight,
               "fc_weight": model.fc.weight, "fc_bias": model.fc.bias}
    for name in ("bn0", "bn1", "bn2"):
        bn = getattr(model, name)
        tensors.update({name + "_weight": bn.weight, name + "_bias": bn.bias,
                        name + "_mean": bn.running_mean, name + "_var": bn.running_var})
    for name in ("conv1", "conv2", "conv3"):
        conv = getattr(model, name)
        tensors.update({name + "_weight": conv.weight, name + "_bias": conv.bias})
    gate = getattr(model, "W_gate_e", None)
    if gate is not None:
        tensors.update({"W_gate_e_weight": gate.weight, "W_gate_e_bias": gate.bias})
    way = "serial" if model.way == "serial" else "parallel"      # the reference's test: any other value is parallel
    p = acre_struct(way, model.in_channels, (model.first_atrous, model.second_atrous, model.third_atrous),
                    model.ent_embeddings.weight.shape[1], model.rel_embeddings.weight.shape[0])
    p.bn0_eps, p.bn1_eps, p.bn2_eps = float(model.bn0.eps), float(model.bn1.eps), float(model.bn2.eps)
    for name in ACRE_FIELDS:
        t = tensors.get(name)
        setattr(p, name, None if t is None else _dev_f32(t.detach(), name).data_ptr())
    if out is None:
        out = torch.empty((Q, int(p.hidden_size)), dtype=torch.float32, device=e.device)
    per_query = int(lib().kge_acre_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(1)))
    if per_query == 0:    # unsupported configuration: the call below reports why
        chunk = max(Q, 1)
    else:
        chunk = max(1, min(max(Q, 1), int(ACRE_WORKSPACE_CAP if cap is None else cap) // per_query))
    nbytes = int(lib().kge_acre_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(chunk)))
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=e.device)
    for q0 in range(0, max(Q, 1), chunk):
        n = min(chunk, Q - q0)
        check(lib().kge_acre_trunk_fwd(ctypes.byref(p), _ptr(e[q0:q0 + n]), _ptr(r[q0:q0 + n]), ctypes.c_int64(n),
                                       _ptr(out[q0:q0 + n]), _ptr(workspace), ctypes.c_int64(workspace.numel()),
                                       _stream()), "kge_acre_trunk_fwd")
    return out


PROJE_FIELDS = ("ent", "rel", "bc1", "De1", "Dr1", "bc2", "De2", "Dr2")   # = ProjE_pointwise.parameter_list


class KgeProje(ctypes.Structure):
    """kge_proje_t of include/kge_b200.h."""
    _fields_ = [("hidden_size", ctypes.c_int32), ("num_ent", ctypes.c_int64), ("num_rel", ctypes.c_int64)] + \
        [(n, ctypes.c_void_p) for n in PROJE_FIELDS]


def proje_struct(tables):
    """a KgeProje over the eight tables in parameter_list order (ent, rel, bc1, De1, Dr1, bc2, De2, Dr2)"""
    tables = [_dev_f32(t.detach(), n) for t, n in zip(tables, PROJE_FIELDS)]
    if len(tables) != 8:
        raise KgeError("ProjE needs its eight tables")
    p = KgeProje()
    p.hidden_size, p.num_ent, p.num_rel = int(tables[0].shape[1]), int(tables[0].shape[0]), int(tables[1].shape[0])
    for n, t in zip(PROJE_FIELDS, tables):
        setattr(p, n, t.data_ptr())
    return p


def proje_trunk_fwd(tables, e, r, direction=0, noise=None, out=None):
    """ProjE f1 (direction 0, tail) / f2 (direction 1, head) for ids e, r -> x [Q,k] (times noise [Q,k] if given)"""
    p = proje_struct(tables)
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    if r.numel() != Q:
        raise KgeError("e and r must have equal length")
    if noise is not None and (_dev_f32(noise, "noise").numel() != Q * p.hidden_size):
        raise KgeError("noise must be [Q, hidden_size]")
    if out is None:
        out = torch.empty((Q, p.hidden_size), dtype=torch.float32, device=e.device)
    check(lib().kge_proje_trunk_fwd(ctypes.byref(p), ctypes.c_int32(direction), _ptr(e), _ptr(r), ctypes.c_int64(Q),
                                    _ptr(noise), _ptr(out), _stream()), "kge_proje_trunk_fwd")
    return out


def proje_train_step(tables, h, r, t, hr_t, tr_h, grads, noise_tail=None, noise_head=None, loss_out=None):
    """ProjE forward + loss + backward of both directions (hr_t or tr_h None: that direction is skipped) in one
    launch.  grads: eight dense buffers shaped like the tables (or None), accumulated.  -> loss [1]"""
    p = proje_struct(tables)
    r = _dev_i64(r, "r")
    B, N, k = r.numel(), p.num_ent, p.hidden_size
    for ids, lab, nz, name in ((h, hr_t, noise_tail, "tail"), (t, tr_h, noise_head, "head")):
        if lab is None:
            continue
        if _dev_i64(ids, "ids").numel() != B or _dev_f32(lab, "labels").shape != (B, N):
            raise KgeError("%s direction: ids [B] and labels [B, num_ent] expected" % name)
        if nz is not None and _dev_f32(nz, "noise").numel() != B * k:
            raise KgeError("%s direction: noise must be [B, hidden_size]" % name)
    if loss_out is None:
        loss_out = torch.empty(1, dtype=torch.float32, device=r.device)
    for g, w in zip(grads, tables):
        if g is not None and (_dev_f32(g, "grad").shape != w.shape):
            raise KgeError("gradient buffers must be shaped like the tables")
    check(lib().kge_proje_train_step(ctypes.byref(p), _ptr(h if hr_t is not None else None), _ptr(r),
                                     _ptr(t if tr_h is not None else None), ctypes.c_int64(B), _ptr(hr_t), _ptr(tr_h),
                                     _ptr(noise_tail if hr_t is not None else None),
                                     _ptr(noise_head if tr_h is not None else None), _table_ptr_array(grads),
                                     _ptr(loss_out), _stream()), "kge_proje_train_step")
    return loss_out


def reg_l1_dense(tensors, grads, lmbda, out=None):
    """lmbda * sum |w| over every element of `tensors` -> [1]; grads (same length, entries may be None; or None)
    += lmbda * sign(w)"""
    ts = [_dev_f32(t.detach(), "w") for t in tensors]
    if len(ts) > MAX_TABLES:
        raise KgeError("at most %d tensors" % MAX_TABLES)
    if out is None:
        out = torch.empty(1, dtype=torch.float32, device=ts[0].device)
    ws = _table_ptr_array(ts)
    gs = _table_ptr_array(grads) if grads is not None else None
    ns = (ctypes.c_int64 * MAX_TABLES)(*[t.numel() for t in ts])
    check(lib().kge_reg_l1_dense(ws, gs, ns, ctypes.c_int32(len(ts)), ctypes.c_float(lmbda), _ptr(out), _stream()),
          "kge_reg_l1_dense")
    return out


def proj_labels_negatives(labels, neg):
    """labels [B,N] (in place): -1 at the distinct entity ids neg wherever the label is still 0"""
    labels, neg = _dev_f32(labels, "labels"), _dev_i64(neg, "neg")
    B, N = labels.shape
    check(lib().kge_proj_labels_negatives(_ptr(labels), ctypes.c_int64(B), ctypes.c_int64(N), _ptr(neg),
                                          ctypes.c_int64(neg.numel()), _stream()), "kge_proj_labels_negatives")
    return labels


# ---- TuckER (include/kge_b200.h: kge_tucker_*) ---------------------------------------------------
TUCKER_FIELDS = ("ent", "rel", "W")   # = TuckER.parameter_list
TUCKER_MASK_NONE, TUCKER_MASK_EXPLICIT, TUCKER_MASK_COUNTER = 0, 1, 2


class KgeTucker(ctypes.Structure):
    """kge_tucker_t of include/kge_b200.h."""
    _fields_ = [("d1", ctypes.c_int32), ("d2", ctypes.c_int32), ("num_ent", ctypes.c_int64),
                ("num_rel", ctypes.c_int64)] + [(n, ctypes.c_void_p) for n in TUCKER_FIELDS]


class KgeTuckerMask(ctypes.Structure):
    """kge_tucker_mask_t of include/kge_b200.h."""
    _fields_ = [("mode", ctypes.c_int32), ("noise1", ctypes.c_void_p), ("seed", ctypes.c_uint64),
                ("offset", ctypes.c_uint64), ("p", ctypes.c_float)]


def tucker_struct(tables):
    """a KgeTucker over (ent [N,d1], rel [R,d2], W [d2,d1*d1])"""
    if len(tables) != 3:
        raise KgeError("TuckER needs its three tables")
    ent, rel, W = [_dev_f32(t.detach(), n) for t, n in zip(tables, TUCKER_FIELDS)]
    if ent.dim() != 2 or rel.dim() != 2 or tuple(W.shape) != (rel.shape[1], ent.shape[1] * ent.shape[1]):
        raise KgeError("TuckER tables must be ent [N,d1], rel [R,d2], W [d2,d1*d1]")
    p = KgeTucker()
    p.d1, p.d2, p.num_ent, p.num_rel = int(ent.shape[1]), int(rel.shape[1]), int(ent.shape[0]), int(rel.shape[0])
    p.ent, p.rel, p.W = ent.data_ptr(), rel.data_ptr(), W.data_ptr()
    return p


def tucker_mask(Q, d1, noise1=None, counter=None):
    """kge_tucker_mask_t (or None): noise1 [Q,d1,d1] for the explicit mode, counter = (seed, offset, p) for the
    counter mode."""
    if noise1 is not None:
        if counter is not None:
            raise KgeError("explicit and counter mask are exclusive")
        if _dev_f32(noise1, "noise1").numel() != Q * d1 * d1:
            raise KgeError("noise1 must be [Q, d1, d1]")
        return KgeTuckerMask(TUCKER_MASK_EXPLICIT, noise1.data_ptr(), 0, 0, 0.0)
    if counter is None:
        return None
    seed, offset, p = counter
    if not 0.0 <= float(p) <= 1.0:
        raise KgeError("dropout probability must be in [0, 1]")
    return KgeTuckerMask(TUCKER_MASK_COUNTER, None, int(seed), int(offset), float(p))


def _tucker_workspace(p, U, device):
    n = int(lib().kge_tucker_workspace_bytes(ctypes.byref(p), ctypes.c_int64(U)))
    return torch.empty(max(n, 16), dtype=torch.uint8, device=device)


def tucker_cores(tables, ids, out=None):
    """M [U, d1*d1]: the core matrix sum_k rel[ids[u], k] W[k] of every relation id in ids (projection.py:321-323,
    once per relation instead of once per sample)"""
    p = tucker_struct(tables)
    ids = _dev_i64(ids, "ids")
    U = ids.numel()
    if out is None:
        out = torch.empty((U, p.d1 * p.d1), dtype=torch.float32, device=ids.device)
    elif _dev_f32(out, "out").numel() != U * p.d1 * p.d1:
        raise KgeError("out must be [U, d1*d1]")
    ws = _tucker_workspace(p, U, ids.device)
    check(lib().kge_tucker_cores(ctypes.byref(p), _ptr(ids), ctypes.c_int64(U), _ptr(out), _ptr(ws),
                                 ctypes.c_int64(ws.numel()), _stream()), "kge_tucker_cores")
    return out


def _tucker_trunk_args(p, M, e, slot, noise0, noise2, noise1, counter):
    M, e, slot = _dev_f32(M, "M"), _dev_i64(e, "e"), _dev_i64(slot, "slot")
    Q = e.numel()
    if slot.numel() != Q:
        raise KgeError("e and slot must have equal length")
    if M.dim() != 2 or M.shape[1] != p.d1 * p.d1:
        raise KgeError("M must be [U, d1*d1]")
    for nz, name in ((noise0, "noise0"), (noise2, "noise2")):
        if nz is not None and _dev_f32(nz, name).numel() != Q * p.d1:
            raise KgeError("%s must be [Q, d1]" % name)
    return M, e, slot, Q, tucker_mask(Q, p.d1, noise1, counter)


def tucker_trunk_fwd(tables, M, e, slot, noise0=None, noise2=None, noise1=None, counter=None, save=False):
    """TuckER's trunk (projection.py:318-328) for entity ids e and core-matrix rows slot -> x [Q,d1], or with
    save=True (x, xpre [Q,d1], nrm [Q]) for tucker_trunk_bwd.  noise1 / counter: see tucker_mask."""
    p = tucker_struct(tables)
    M, e, slot, Q, mask = _tucker_trunk_args(p, M, e, slot, noise0, noise2, noise1, counter)
    x = torch.empty((Q, p.d1), dtype=torch.float32, device=e.device)
    xpre = torch.empty_like(x) if save else None
    nrm = torch.empty(Q, dtype=torch.float32, device=e.device) if save else None
    check(lib().kge_tucker_trunk_fwd(ctypes.byref(p), _ptr(M), _ptr(e), _ptr(slot), ctypes.c_int64(Q), _ptr(noise0),
                                     ctypes.byref(mask) if mask is not None else None, _ptr(noise2), _ptr(x),
                                     _ptr(xpre), _ptr(nrm), _stream()), "kge_tucker_trunk_fwd")
    return (x, xpre, nrm) if save else x


def tucker_trunk_bwd(tables, M, e, slot, gx, xpre, nrm, grad_ent=None, dM=None, noise0=None, noise2=None, noise1=None,
                     counter=None):
    """backward of tucker_trunk_fwd: accumulates into grad_ent [N,d1] and dM [U,d1*d1] (each may be None)"""
    p = tucker_struct(tables)
    M, e, slot, Q, mask = _tucker_trunk_args(p, M, e, slot, noise0, noise2, noise1, counter)
    if _dev_f32(gx, "gx").numel() != Q * p.d1 or _dev_f32(xpre, "xpre").numel() != Q * p.d1 or \
            _dev_f32(nrm, "nrm").numel() != Q:
        raise KgeError("gx and xpre must be [Q, d1], nrm [Q]")
    if grad_ent is not None and _dev_f32(grad_ent, "grad_ent").shape != tables[0].shape:
        raise KgeError("grad_ent must be shaped like the entity table")
    if dM is not None and _dev_f32(dM, "dM").shape != M.shape:
        raise KgeError("dM must be shaped like M")
    check(lib().kge_tucker_trunk_bwd(ctypes.byref(p), _ptr(M), _ptr(e), _ptr(slot), ctypes.c_int64(Q), _ptr(noise0),
                                     ctypes.byref(mask) if mask is not None else None, _ptr(noise2), _ptr(gx),
                                     _ptr(xpre), _ptr(nrm), _ptr(grad_ent), _ptr(dM), _stream()),
          "kge_tucker_trunk_bwd")


def tucker_cores_bwd(tables, ids, dM, grad_rel=None, grad_W=None):
    """backward of tucker_cores: accumulates into grad_rel [R,d2] and grad_W [d2,d1*d1] (each may be None)"""
    p = tucker_struct(tables)
    ids = _dev_i64(ids, "ids")
    U = ids.numel()
    if _dev_f32(dM, "dM").numel() != U * p.d1 * p.d1:
        raise KgeError("dM must be [U, d1*d1]")
    for g, w in ((grad_rel, tables[1]), (grad_W, tables[2])):
        if g is not None and _dev_f32(g, "grad").shape != w.shape:
            raise KgeError("gradient buffers must be shaped like the tables")
    ws = _tucker_workspace(p, U, ids.device)
    check(lib().kge_tucker_cores_bwd(ctypes.byref(p), _ptr(ids), ctypes.c_int64(U), _ptr(dM), _ptr(grad_rel),
                                     _ptr(grad_W), _ptr(ws), ctypes.c_int64(ws.numel()), _stream()),
          "kge_tucker_cores_bwd")


def tucker_mask1(seed, offset, p, Q, d1, device="cuda"):
    """the counter-mode dropout1 mask of (seed, offset, p) as a [Q, d1, d1] float tensor"""
    out = torch.empty((Q, d1, d1), dtype=torch.float32, device=device)
    check(lib().kge_tucker_mask1(ctypes.c_uint64(int(seed)), ctypes.c_uint64(int(offset)), ctypes.c_float(p),
                                 ctypes.c_int64(Q), ctypes.c_int32(d1), _ptr(out), _stream()), "kge_tucker_mask1")
    return out


# ---- ConvE training-mode trunk (include/kge_b200.h: kge_conve_train_*) ------------------------------------------
CONVE_TRAIN_PARAMS = ("ent", "rel", "bn0_weight", "bn0_bias", "conv_weight", "conv_bias", "bn1_weight", "bn1_bias",
                      "fc_weight", "fc_bias", "bn2_weight", "bn2_bias")   # = the gradient order of kge_conve_train_bwd
CONVE_TRAIN_RUNNING = ("bn0_mean", "bn0_var", "bn1_mean", "bn1_var", "bn2_mean", "bn2_var")


class KgeConveTrain(ctypes.Structure):
    """kge_conve_train_t of include/kge_b200.h."""
    _fields_ = [("hidden_size", ctypes.c_int32), ("hidden_size_1", ctypes.c_int32)] + \
               [(n, ctypes.c_float) for n in ("bn0_eps", "bn1_eps", "bn2_eps", "bn0_momentum", "bn1_momentum",
                                              "bn2_momentum")] + \
               [(n, ctypes.c_void_p) for n in CONVE_TRAIN_PARAMS + CONVE_TRAIN_RUNNING]


def conve_train_struct(model, params=None, running=True):
    """kge_conve_train_t of a ConvE (the reference's sub-module names).  params: the 12 tensors of CONVE_TRAIN_PARAMS
    (default: the model's own); running=False leaves the running statistics alone (NULL pointers)."""
    if params is None:
        params = model.kge_conve_params()
    if len(params) != len(CONVE_TRAIN_PARAMS):
        raise KgeError("ConvE's training trunk needs its %d parameter tensors" % len(CONVE_TRAIN_PARAMS))
    p = KgeConveTrain()
    p.hidden_size, p.hidden_size_1 = int(model.hidden_size), int(model.hidden_size_1)
    bns = (model.bn0, model.bn1, model.bn2)
    p.bn0_eps, p.bn1_eps, p.bn2_eps = (float(bn.eps) for bn in bns)
    if any(bn.momentum is None for bn in bns):   # cumulative averaging: the torch layers' job
        raise KgeNotSupported("kge_conve_train: BatchNorm momentum None is not supported")
    p.bn0_momentum, p.bn1_momentum, p.bn2_momentum = (float(bn.momentum) for bn in bns)
    for name, t in zip(CONVE_TRAIN_PARAMS, params):
        setattr(p, name, _dev_f32(t.detach(), name).data_ptr())
    if running:
        for i, bn in enumerate(bns):
            setattr(p, "bn%d_mean" % i, _dev_f32(bn.running_mean, "running_mean").data_ptr())
            setattr(p, "bn%d_var" % i, _dev_f32(bn.running_var, "running_var").data_ptr())
    return p


def _conve_train_noise(noise, rows, width, name):
    if noise is not None and (_dev_f32(noise, name).numel() != rows * width):
        raise KgeError("%s must be [Q, %d]" % (name, width))
    return _ptr(noise)


def conve_train_fwd(model, e, r, B, noise0=None, noise1=None, noise2=None, params=None, running=True):
    """ConvE's trunk in training mode (projection.py:86-99) on Q = G * B rows, G groups of B with their own batch
    statistics -> (x [Q, k], workspace).  Updates the model's running statistics in place (group after group) unless
    running=False; num_batches_tracked is the caller's.  Keep the workspace for conve_train_bwd."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    if r.numel() != Q:
        raise KgeError("e and r must have equal length")
    p = conve_train_struct(model, params, running)
    k = p.hidden_size
    n0 = _conve_train_noise(noise0, Q, 2 * k, "noise0")
    n1 = _conve_train_noise(noise1, Q, 32, "noise1")
    n2 = _conve_train_noise(noise2, Q, k, "noise2")
    nbytes = int(lib().kge_conve_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q), ctypes.c_int64(B)))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=e.device)
    x = torch.empty((Q, k), dtype=torch.float32, device=e.device)
    check(lib().kge_conve_train_fwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), ctypes.c_int64(B), n0, n1,
                                    n2, _ptr(x), _ptr(ws), ctypes.c_int64(ws.numel()), _stream()),
          "kge_conve_train_fwd")
    return x, ws


def conve_train_bwd(model, e, r, B, gx, x, grads, workspace, noise0=None, noise1=None, noise2=None, params=None):
    """backward of conve_train_fwd: accumulates into grads, 12 buffers shaped like CONVE_TRAIN_PARAMS"""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    p = conve_train_struct(model, params, running=False)
    params = params if params is not None else model.kge_conve_params()
    k = p.hidden_size
    if _dev_f32(gx, "gx").numel() != Q * k or _dev_f32(x, "x").numel() != Q * k:
        raise KgeError("gx and x must be [Q, k]")
    if len(grads) != len(CONVE_TRAIN_PARAMS) or any(_dev_f32(g, "grad").shape != w.shape for g, w in zip(grads, params)):
        raise KgeError("grads must be %d buffers shaped like the parameters" % len(CONVE_TRAIN_PARAMS))
    n0 = _conve_train_noise(noise0, Q, 2 * k, "noise0")
    n1 = _conve_train_noise(noise1, Q, 32, "noise1")
    n2 = _conve_train_noise(noise2, Q, k, "noise2")
    arr = (ctypes.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
    check(lib().kge_conve_train_bwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), ctypes.c_int64(B), n0, n1,
                                    n2, _ptr(gx), _ptr(x), arr, _ptr(workspace), ctypes.c_int64(workspace.numel()),
                                    _stream()), "kge_conve_train_bwd")


# ---- HypER training-mode trunk (include/kge_b200.h: kge_hyper_train_*) ------------------------------------------
HYPER_TRAIN_PARAMS = ("ent", "rel", "bn0_weight", "bn0_bias", "bn1_weight", "bn1_bias", "fc_weight", "fc_bias",
                      "bn2_weight", "bn2_bias", "fc1_weight", "fc1_bias")   # = the gradient order of kge_hyper_train_bwd
HYPER_TRAIN_RUNNING = CONVE_TRAIN_RUNNING


class KgeHyperTrain(ctypes.Structure):
    """kge_hyper_train_t of include/kge_b200.h."""
    _fields_ = [("ent_hidden_size", ctypes.c_int32), ("rel_hidden_size", ctypes.c_int32),
                ("ent_padding_idx", ctypes.c_int64), ("rel_padding_idx", ctypes.c_int64)] + \
               [(n, ctypes.c_float) for n in ("bn0_eps", "bn1_eps", "bn2_eps", "bn0_momentum", "bn1_momentum",
                                              "bn2_momentum")] + \
               [(n, ctypes.c_void_p) for n in HYPER_TRAIN_PARAMS + HYPER_TRAIN_RUNNING]


def hyper_train_struct(model, params=None, running=True):
    """kge_hyper_train_t of a HypER (the reference's sub-module names).  params: the 12 tensors of HYPER_TRAIN_PARAMS
    (default: model.kge_hyper_params()); running=False leaves the running statistics alone (NULL pointers)."""
    if params is None:
        params = model.kge_hyper_params()
    if len(params) != len(HYPER_TRAIN_PARAMS):
        raise KgeError("HypER's training trunk needs its %d parameter tensors" % len(HYPER_TRAIN_PARAMS))
    p = KgeHyperTrain()
    p.ent_hidden_size, p.rel_hidden_size = int(model.ent_hidden_size), int(model.rel_hidden_size)
    pads = (model.ent_embeddings.padding_idx, model.rel_embeddings.padding_idx)
    p.ent_padding_idx, p.rel_padding_idx = (-1 if i is None else int(i) for i in pads)
    bns = (model.bn0, model.bn1, model.bn2)
    p.bn0_eps, p.bn1_eps, p.bn2_eps = (float(bn.eps) for bn in bns)
    if any(bn.momentum is None for bn in bns):   # cumulative averaging: the torch layers' job
        raise KgeNotSupported("kge_hyper_train: BatchNorm momentum None is not supported")
    p.bn0_momentum, p.bn1_momentum, p.bn2_momentum = (float(bn.momentum) for bn in bns)
    for name, t in zip(HYPER_TRAIN_PARAMS, params):
        setattr(p, name, _dev_f32(t.detach(), name).data_ptr())
    if running:
        for i, bn in enumerate(bns):
            setattr(p, "bn%d_mean" % i, _dev_f32(bn.running_mean, "running_mean").data_ptr())
            setattr(p, "bn%d_var" % i, _dev_f32(bn.running_var, "running_var").data_ptr())
    return p


def hyper_train_fwd(model, e, r, B, noise0=None, noise1=None, noise2=None, params=None, running=True):
    """HypER's trunk in training mode (projection.py:581-606) on Q = G * B rows, G groups of B with their own batch
    statistics -> (x [Q, de], workspace).  Updates the model's running statistics in place (group after group) unless
    running=False; num_batches_tracked is the caller's.  Keep the workspace for hyper_train_bwd."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    if r.numel() != Q:
        raise KgeError("e and r must have equal length")
    p = hyper_train_struct(model, params, running)
    de = p.ent_hidden_size
    n0 = _conve_train_noise(noise0, Q, de, "noise0")
    n1 = _conve_train_noise(noise1, Q, 32, "noise1")
    n2 = _conve_train_noise(noise2, Q, de, "noise2")
    nbytes = int(lib().kge_hyper_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q), ctypes.c_int64(B)))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=e.device)
    x = torch.empty((Q, de), dtype=torch.float32, device=e.device)
    check(lib().kge_hyper_train_fwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), ctypes.c_int64(B), n0, n1,
                                    n2, _ptr(x), _ptr(ws), ctypes.c_int64(ws.numel()), _stream()),
          "kge_hyper_train_fwd")
    return x, ws


def hyper_train_bwd(model, e, r, B, gx, x, grads, workspace, noise0=None, noise1=None, noise2=None, params=None):
    """backward of hyper_train_fwd: accumulates into grads, 12 buffers shaped like HYPER_TRAIN_PARAMS"""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    p = hyper_train_struct(model, params, running=False)
    params = params if params is not None else model.kge_hyper_params()
    de = p.ent_hidden_size
    if _dev_f32(gx, "gx").numel() != Q * de or _dev_f32(x, "x").numel() != Q * de:
        raise KgeError("gx and x must be [Q, de]")
    if len(grads) != len(HYPER_TRAIN_PARAMS) or any(_dev_f32(g, "grad").shape != w.shape for g, w in zip(grads, params)):
        raise KgeError("grads must be %d buffers shaped like the parameters" % len(HYPER_TRAIN_PARAMS))
    n0 = _conve_train_noise(noise0, Q, de, "noise0")
    n1 = _conve_train_noise(noise1, Q, 32, "noise1")
    n2 = _conve_train_noise(noise2, Q, de, "noise2")
    arr = (ctypes.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
    check(lib().kge_hyper_train_bwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), ctypes.c_int64(B), n0, n1,
                                    n2, _ptr(gx), _ptr(x), arr, _ptr(workspace), ctypes.c_int64(workspace.numel()),
                                    _stream()), "kge_hyper_train_bwd")


# ---- InteractE training-mode trunk (include/kge_b200.h: kge_interacte_train_*) --------------------------------------
INTERACTE_TRAIN_PARAMS = ("ent", "rel", "bn0_weight", "bn0_bias", "conv_filt", "bn1_weight", "bn1_bias", "fc_weight",
                          "fc_bias", "bn2_weight", "bn2_bias")   # = the gradient order of kge_interacte_train_bwd
INTERACTE_TRAIN_RUNNING = CONVE_TRAIN_RUNNING


class KgeInteracteTrain(ctypes.Structure):
    """kge_interacte_train_t of include/kge_b200.h."""
    _fields_ = [(n, ctypes.c_int32) for n in ("feature_permutation", "num_filters", "kernel_size", "reshape_height",
                                              "reshape_width")] + \
               [(n, ctypes.c_float) for n in ("bn0_eps", "bn1_eps", "bn2_eps", "bn0_momentum", "bn1_momentum",
                                              "bn2_momentum")] + \
               [("perm", ctypes.c_void_p)] + \
               [(n, ctypes.c_void_p) for n in INTERACTE_TRAIN_PARAMS + INTERACTE_TRAIN_RUNNING]


def interacte_train_struct(model, params=None, running=True, perm=None):
    """kge_interacte_train_t of an InteractE (the reference's sub-module names).  params: the 11 tensors of
    INTERACTE_TRAIN_PARAMS (default: model.kge_interacte_params()); running=False leaves the running statistics alone
    (NULL pointers); perm: the chequer permutation, int64 on the tables' device (default: model.chequer_perm)."""
    if params is None:
        params = model.kge_interacte_params()
    if len(params) != len(INTERACTE_TRAIN_PARAMS):
        raise KgeError("InteractE's training trunk needs its %d parameter tensors" % len(INTERACTE_TRAIN_PARAMS))
    p = KgeInteracteTrain()
    p.feature_permutation, p.num_filters, p.kernel_size = (int(model.feature_permutation), int(model.num_filters),
                                                           int(model.kernel_size))
    p.reshape_height, p.reshape_width = int(model.reshape_height), int(model.reshape_width)
    bns = (model.bn0, model.bn1, model.bn2)
    p.bn0_eps, p.bn1_eps, p.bn2_eps = (float(bn.eps) for bn in bns)
    if any(bn.momentum is None for bn in bns):   # cumulative averaging: the torch layers' job
        raise KgeNotSupported("kge_interacte_train: BatchNorm momentum None is not supported")
    p.bn0_momentum, p.bn1_momentum, p.bn2_momentum = (float(bn.momentum) for bn in bns)
    for name, t in zip(INTERACTE_TRAIN_PARAMS, params):
        setattr(p, name, _dev_f32(t.detach(), name).data_ptr())
    perm = model.chequer_perm if perm is None else perm
    if perm.device != params[0].device or perm.dtype != torch.int64:
        perm = perm.to(device=params[0].device, dtype=torch.int64)
    p.perm = _dev_i64(perm.contiguous(), "chequer_perm").data_ptr()
    if running:
        for i, bn in enumerate(bns):
            setattr(p, "bn%d_mean" % i, _dev_f32(bn.running_mean, "running_mean").data_ptr())
            setattr(p, "bn%d_var" % i, _dev_f32(bn.running_var, "running_var").data_ptr())
    return p, perm


def _interacte_noise_widths(p):
    """(noise0, noise1, noise2) row widths: P * 2k, P * F, k"""
    k = p.reshape_height * p.reshape_width
    return p.feature_permutation * 2 * k, p.feature_permutation * p.num_filters, k


def interacte_train_workspace_bytes(model, Q, B):
    """bytes of device workspace one kge_interacte_train_fwd / _bwd pair needs for Q = G * B rows (0 for a geometry
    the kernels refuse)"""
    p = KgeInteracteTrain()
    p.feature_permutation, p.num_filters, p.kernel_size = (int(model.feature_permutation), int(model.num_filters),
                                                           int(model.kernel_size))
    p.reshape_height, p.reshape_width = int(model.reshape_height), int(model.reshape_width)
    return int(lib().kge_interacte_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q), ctypes.c_int64(B)))


def interacte_train_fwd(model, e, r, B, noise0=None, noise1=None, noise2=None, params=None, running=True, perm=None):
    """InteractE's trunk in training mode (projection.py:425-442) on Q = G * B rows, G groups of B with their own batch
    statistics -> (x [Q, k], workspace).  Updates the model's running statistics in place (group after group) unless
    running=False; num_batches_tracked is the caller's.  Keep the workspace for ONE interacte_train_bwd."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    if r.numel() != Q:
        raise KgeError("e and r must have equal length")
    p, perm = interacte_train_struct(model, params, running, perm)
    w0, w1, w2 = _interacte_noise_widths(p)
    n0 = _conve_train_noise(noise0, Q, w0, "noise0")
    n1 = _conve_train_noise(noise1, Q, w1, "noise1")
    n2 = _conve_train_noise(noise2, Q, w2, "noise2")
    nbytes = int(lib().kge_interacte_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q), ctypes.c_int64(B)))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=e.device)
    x = torch.empty((Q, w2), dtype=torch.float32, device=e.device)
    check(lib().kge_interacte_train_fwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), ctypes.c_int64(B), n0,
                                        n1, n2, _ptr(x), _ptr(ws), ctypes.c_int64(ws.numel()), _stream()),
          "kge_interacte_train_fwd")
    return x, ws


def interacte_train_bwd(model, e, r, B, gx, x, grads, workspace, noise0=None, noise1=None, noise2=None, params=None,
                        perm=None):
    """backward of interacte_train_fwd: accumulates into grads, 11 buffers shaped like INTERACTE_TRAIN_PARAMS.  It
    overwrites the forward's feature maps in the workspace: one backward per forward."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    params = params if params is not None else model.kge_interacte_params()
    p, perm = interacte_train_struct(model, params, False, perm)
    w0, w1, w2 = _interacte_noise_widths(p)
    if _dev_f32(gx, "gx").numel() != Q * w2 or _dev_f32(x, "x").numel() != Q * w2:
        raise KgeError("gx and x must be [Q, k]")
    if len(grads) != len(INTERACTE_TRAIN_PARAMS) or \
            any(_dev_f32(g, "grad").shape != w.shape for g, w in zip(grads, params)):
        raise KgeError("grads must be %d buffers shaped like the parameters" % len(INTERACTE_TRAIN_PARAMS))
    n0 = _conve_train_noise(noise0, Q, w0, "noise0")
    n1 = _conve_train_noise(noise1, Q, w1, "noise1")
    n2 = _conve_train_noise(noise2, Q, w2, "noise2")
    arr = (ctypes.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
    check(lib().kge_interacte_train_bwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), ctypes.c_int64(B), n0,
                                        n1, n2, _ptr(gx), _ptr(x), arr, _ptr(workspace),
                                        ctypes.c_int64(workspace.numel()), _stream()), "kge_interacte_train_bwd")


# ---- AcrE training-mode trunk (include/kge_b200.h: kge_acre_train_*) ----------------------------------------------
ACRE_TRAIN_PARAMS = ("ent", "rel", "bn0_weight", "bn0_bias", "conv1_weight", "conv1_bias", "conv2_weight",
                     "conv2_bias", "conv3_weight", "conv3_bias", "W_gate_e_weight", "W_gate_e_bias", "bn1_weight",
                     "bn1_bias", "fc_weight", "fc_bias", "bn2_weight", "bn2_bias")   # = kge_acre_train_bwd's slots
ACRE_TRAIN_RUNNING = CONVE_TRAIN_RUNNING


class KgeAcreTrain(ctypes.Structure):
    """kge_acre_train_t of include/kge_b200.h."""
    _fields_ = [(n, ctypes.c_int32) for n in ("in_channels", "way", "first_atrous", "second_atrous", "third_atrous",
                                              "hidden_size")] + \
               [("num_rel", ctypes.c_int64)] + \
               [(n, ctypes.c_float) for n in ("bn0_eps", "bn1_eps", "bn2_eps", "bn0_momentum", "bn1_momentum",
                                              "bn2_momentum")] + \
               [(n, ctypes.c_void_p) for n in ACRE_TRAIN_PARAMS + ACRE_TRAIN_RUNNING]


def acre_train_present(model):
    """the names of ACRE_TRAIN_PARAMS this AcrE has: no conv biases without acre_bias, W_gate_e in the parallel way
    only"""
    par = model.way != "serial"
    bias = model.conv1.bias is not None
    return tuple(n for n in ACRE_TRAIN_PARAMS
                 if not (n.startswith("conv") and n.endswith("_bias") and not bias)
                 and not (n.startswith("W_gate_e") and not par))


def _acre_train_config(model):
    p = KgeAcreTrain()
    way = "serial" if model.way == "serial" else "parallel"      # the reference's test: any other value is parallel
    p.way = ACRE_WAYS[way]
    p.in_channels, p.hidden_size = int(model.in_channels), int(model.ent_embeddings.weight.shape[1])
    p.num_rel = int(model.rel_embeddings.weight.shape[0])
    p.first_atrous, p.second_atrous, p.third_atrous = (int(model.first_atrous), int(model.second_atrous),
                                                       int(model.third_atrous))
    return p


def acre_train_struct(model, params=None, running=True):
    """kge_acre_train_t of an AcrE (the reference's sub-module names).  params: the present trunk tensors in
    ACRE_TRAIN_PARAMS order (default: model.kge_acre_params()); running=False leaves the running statistics alone
    (NULL pointers).  Absent parameters stay NULL."""
    if params is None:
        params = model.kge_acre_params()
    names = acre_train_present(model)
    if len(params) != len(names):
        raise KgeError("AcrE's training trunk needs its %d parameter tensors" % len(names))
    p = _acre_train_config(model)
    bns = (model.bn0, model.bn1, model.bn2)
    p.bn0_eps, p.bn1_eps, p.bn2_eps = (float(bn.eps) for bn in bns)
    if any(bn.momentum is None for bn in bns):   # cumulative averaging: the torch layers' job
        raise KgeNotSupported("kge_acre_train: BatchNorm momentum None is not supported")
    p.bn0_momentum, p.bn1_momentum, p.bn2_momentum = (float(bn.momentum) for bn in bns)
    for name, t in zip(names, params):
        setattr(p, name, _dev_f32(t.detach(), name).data_ptr())
    if running:
        for i, bn in enumerate(bns):
            setattr(p, "bn%d_mean" % i, _dev_f32(bn.running_mean, "running_mean").data_ptr())
            setattr(p, "bn%d_var" % i, _dev_f32(bn.running_var, "running_var").data_ptr())
    return p


def acre_train_workspace_bytes(model, Q, B):
    """bytes of device workspace one kge_acre_train_fwd / _bwd pair needs for Q = G * B rows (0 for a configuration
    the kernels refuse)"""
    p = _acre_train_config(model)
    return int(lib().kge_acre_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q), ctypes.c_int64(B)))


def acre_train_fwd(model, e, r, B, noise0=None, noise1=None, noise2=None, params=None, running=True):
    """AcrE's trunk in training mode (projection.py:706-734) on Q = G * B rows, G groups of B with their own batch
    statistics -> (x [Q, 200], workspace).  Updates the model's running statistics in place (group after group) unless
    running=False; num_batches_tracked is the caller's.  Keep the workspace for ONE acre_train_bwd."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    if r.numel() != Q:
        raise KgeError("e and r must have equal length")
    p = acre_train_struct(model, params, running)
    n0 = _conve_train_noise(noise0, Q, 400, "noise0")
    n1 = _conve_train_noise(noise1, Q, int(p.in_channels), "noise1")
    n2 = _conve_train_noise(noise2, Q, 200, "noise2")
    nbytes = int(lib().kge_acre_train_workspace_bytes(ctypes.byref(p), ctypes.c_int64(Q), ctypes.c_int64(B)))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=e.device)
    x = torch.empty((Q, 200), dtype=torch.float32, device=e.device)
    check(lib().kge_acre_train_fwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), ctypes.c_int64(B), n0, n1,
                                   n2, _ptr(x), _ptr(ws), ctypes.c_int64(ws.numel()), _stream()), "kge_acre_train_fwd")
    return x, ws


def acre_train_bwd(model, e, r, B, gx, x, grads, workspace, noise0=None, noise1=None, noise2=None, params=None):
    """backward of acre_train_fwd: accumulates into grads, one buffer shaped like each tensor of params (the present
    parameters in ACRE_TRAIN_PARAMS order).  It overwrites the forward's features in the workspace: one backward per
    forward."""
    e, r = _dev_i64(e, "e"), _dev_i64(r, "r")
    Q = e.numel()
    params = params if params is not None else model.kge_acre_params()
    p = acre_train_struct(model, params, False)
    if _dev_f32(gx, "gx").numel() != Q * 200 or _dev_f32(x, "x").numel() != Q * 200:
        raise KgeError("gx and x must be [Q, 200]")
    if len(grads) != len(params) or any(_dev_f32(g, "grad").shape != w.shape for g, w in zip(grads, params)):
        raise KgeError("grads must be %d buffers shaped like the parameters" % len(params))
    n0 = _conve_train_noise(noise0, Q, 400, "noise0")
    n1 = _conve_train_noise(noise1, Q, int(p.in_channels), "noise1")
    n2 = _conve_train_noise(noise2, Q, 200, "noise2")
    slots = dict(zip(acre_train_present(model), grads))
    arr = (ctypes.c_void_p * len(ACRE_TRAIN_PARAMS))(*[slots[n].data_ptr() if n in slots else None
                                                        for n in ACRE_TRAIN_PARAMS])
    check(lib().kge_acre_train_bwd(ctypes.byref(p), _ptr(e), _ptr(r), ctypes.c_int64(Q), ctypes.c_int64(B), n0, n1,
                                   n2, _ptr(gx), _ptr(x), arr, _ptr(workspace), ctypes.c_int64(workspace.numel()),
                                   _stream()), "kge_acre_train_bwd")


def launch_count():
    return int(lib().kge_launch_count())
