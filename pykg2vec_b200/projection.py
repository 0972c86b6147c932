"""Projection models — same surface as pykg2vec/models/projection.py.

ConvE (projection.py:12-125).  The reference's hot spot for these models is the last layer,
`sigmoid(x . E^T + b)` against ALL entities, its BCE loss over the dense [b, N] label matrix
and — at evaluation — one such forward plus a full `topk` per query and direction.  Those are
the hand-written kernels here (include/kge_b200.h kge_proj_*): forward() ends in
ProjTailFunction, the loss is Criterion.multi_class_bce -> kge_proj_bce, and the Evaluator ranks
batches of queries with kge_proj_rank (counts only, no [Q, N] matrix, no sort).

The trunk in front of it (BatchNorm -> 3x3 conv -> BatchNorm -> ReLU -> Linear -> BatchNorm ->
ReLU on a [b, 1, 2*h2, h1] image) runs in two ways:
  * training (BatchNorm batch statistics, dropout): ConveTrunkFunction over kge_conve_train_fwd / _bwd —
    statistics reduced in a fixed order, the running statistics updated in place, dropout as explicit
    noise tensors drawn from torch's generator — or the Trainer's fused step on the same kernels.  The
    reference's torch layers stay as _trunk_layers (TF32 convolutions disabled in forward and backward so
    they stay fp32 like the reference's CPU path): the tests' yardstick, and the path for CPU tables,
    images the kernels refuse and kge_trunk = False;
  * evaluation (`proj_query`, used by the batched Evaluator): kge_conve_trunk_fwd — gather +
    BN0 + conv + BN1 + ReLU in one kernel and the Linear layer through the same tiled GEMM as the
    tail.

HypER (projection.py:508-618) has the same tail and loss; its trunk convolves the BatchNormed entity
row with 32 filters of width 9 that a Linear layer (fc1) generates from the query's relation.  Training
with CUDA tables runs HyperTrunkFunction over kge_hyper_train_fwd / _bwd (the queries' filters on the tiled
GEMM, batch statistics reduced in a fixed order, dropout as explicit noise tensors) or the Trainer's fused
step on the same kernels; the reference's layers (the per-query filters as one grouped convolution, TF32
off) stay as _trunk_layers for CPU tables, widths the kernels refuse, BatchNorms without a momentum or
running statistics, and kge_trunk = False.  Evaluation without autograd runs kge_hyper_trunk_fwd — one GEMM
for every relation's filters, one kernel for gather + bn0 + conv + bn1, the Linear layer on the tail's tiled
GEMM, then bn2 + ReLU.

InteractE (projection.py:347-505) has the same tail and loss; its trunk stacks P chequer-permuted images of the
entity and relation features and convolves them circularly with one shared filter bank.  Training with CUDA tables
runs InteracteTrunkFunction over kge_interacte_train_fwd / _bwd (the circular conv with the filter bank in shared
memory, batch statistics reduced in a fixed order, dropout as explicit noise tensors) or the Trainer's fused step on
the same kernels; the reference's layers (the circular convolution through _Fp32Conv2d, TF32 off) stay as
_trunk_layers for CPU tables, geometries the kernels refuse, BatchNorms without a momentum or running statistics, a
chequer_perm whose rows are not permutations, and kge_trunk = False.  Evaluation without autograd runs
kge_interacte_trunk_fwd — one kernel for gather + permutation + bn0 + circular conv + bn1 + ReLU, then HypER's
Linear GEMM and bn2 + ReLU.

AcrE (projection.py:621-746) has the same tail and loss; its trunk runs three dilated (atrous) 3x3 convolutions
on the 20 x 20 image of the stacked entity and relation rows, chained with a residual add (serial way) or side
by side and mixed per channel by a Linear gate (parallel way).  Training with CUDA tables runs AcreTrunkFunction over
kge_acre_train_fwd / _bwd (the convolutions blocked in shared memory and registers, W_gate_e on the tiled GEMM, batch
statistics reduced in a fixed order, dropout as explicit noise tensors) or the Trainer's fused step on the same
kernels; the reference's layers stay as _trunk_layers for CPU tables, configurations the kernels refuse, BatchNorms
without a momentum or running statistics, and kge_trunk = False.  Evaluation without autograd runs kge_acre_trunk_fwd — one kernel for gather + bn0 + the three convs (+ residual
+ bn1 + ReLU in the serial way; the gate input in the parallel way, then the gate on the tiled GEMM and bn1 +
ReLU), then HypER's Linear GEMM and bn2 + ReLU.

TuckER (projection.py:258-345) has the same tail and loss without a bias row; its trunk contracts the normalised
entity row with a d1 x d1 core matrix that the relation selects from the core tensor W.  The reference builds that
matrix per sample; kge_tucker_cores builds it once per distinct relation and kge_tucker_trunk_fwd / _bwd apply the
dropout on it from a counter, in training (TuckerTrunkFunction, or the Trainer's fused step) and in evaluation
(proj_query_cores: one set of matrices per Evaluator.rank_triples call).

ProjE_pointwise (projection.py:128-257) has no bias row and no BatchNorm: its trunk is tanh(e * De + r * Dr + bc),
and forward() returns the loss itself (-log sigmoid at the positive labels, -log(1 - sigmoid) at the negative
ones, zero-label entities weighted 0).  forward() is one autograd Function over kge_proje_train_step, which scores
only the labelled entries of each row; the batched Evaluator ranks kge_proje_trunk_fwd's x with kge_proj_rank.
"""
import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .criterion import Criterion
from .Domain import NamedEmbedding
from .functional import ProjTailFunction, _require_cuda
from .KGMeta import ProjectionModel


class _Fp32Conv2d(torch.autograd.Function):
    """conv2d whose forward AND backward run with TF32 convolutions disabled: the reference's
    numbers are the fp32 CPU path's, and cuDNN would otherwise round operands to 10-bit
    mantissas (torch.backends.cudnn.allow_tf32 defaults to True).  A context manager around the
    forward call alone would not cover the backward pass, which runs later inside
    loss.backward()."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, dilation, groups):
        ctx.save_for_backward(x, weight)
        ctx.conf = (stride, padding, dilation, groups, bias is not None)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            return torch.nn.functional.conv2d(x, weight, bias, stride, padding, dilation, groups)

    @staticmethod
    def backward(ctx, gout):
        x, weight = ctx.saved_tensors
        stride, padding, dilation, groups, has_bias = ctx.conf
        mask = [ctx.needs_input_grad[0], ctx.needs_input_grad[1], has_bias and ctx.needs_input_grad[2]]
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            gx, gw, gb = torch.ops.aten.convolution_backward(
                gout.contiguous(), x, weight, [weight.shape[0]] if has_bias else None, list(stride),
                list(padding), list(dilation), False, [0, 0], groups, mask)
        return gx, gw, gb, None, None, None, None


def _conv2d_fp32(conv, x):
    return _Fp32Conv2d.apply(x, conv.weight, conv.bias, conv.stride, conv.padding, conv.dilation, conv.groups)


class ConveTrunkFunction(torch.autograd.Function):
    """x = ConvE's trunk in training mode (projection.py:86-99) on kge_conve_train_fwd; backward runs
    kge_conve_train_bwd.  The Q = G * B rows are G groups of B rows, each with its own batch statistics; the forward
    updates the model's running statistics in place (num_batches_tracked is the caller's).  noise0 / noise1 /
    noise2: the dropout noise [Q, 2k] / [Q, 32] / [Q, k], or None.  params: ConvE.kge_conve_params()."""

    @staticmethod
    def forward(ctx, model, e, r, B, noise0, noise1, noise2, *params):
        _require_cuda(e, r, *params)
        params = [t.detach() for t in params]
        e, r = e.contiguous(), r.contiguous()
        x, ws = _lib.conve_train_fwd(model, e, r, B, noise0, noise1, noise2, params=params)
        ctx.model, ctx.B, ctx.noise = model, B, (noise0, noise1, noise2)
        ctx.save_for_backward(e, r, x, ws, *params)
        return x

    @staticmethod
    def backward(ctx, gx):
        e, r, x, ws, *params = ctx.saved_tensors
        grads = [torch.zeros_like(t) for t in params]
        _lib.conve_train_bwd(ctx.model, e, r, ctx.B, gx.contiguous(), x, grads, ws, *ctx.noise, params=params)
        return (None,) * 7 + tuple(g if need else None for g, need in zip(grads, ctx.needs_input_grad[7:]))


class ConvE(ProjectionModel):
    """pykg2vec/models/projection.py:12-125 — same kwargs, sub-module names (state_dict keys
    ent_embeddings / rel_embeddings / b / bn0 / conv2d_1 / bn1 / fc / bn2), parameter_list and
    loss binding.

    In training mode with the tables on a CUDA device the trunk is ConveTrunkFunction (kge_conve_train_*); the
    reference's torch layers stay as _trunk_layers: the yardstick of the tests, the path for CPU tables, for images
    the kernels refuse (2k > 4096) and, with the attribute / kwarg kge_trunk = False, for everything."""

    def __init__(self, **kwargs):
        super(ConvE, self).__init__(self.__class__.__name__.lower())
        param_list = ["tot_entity", "tot_relation", "hidden_size", "hidden_size_1",
                      "lmbda", "input_dropout", "feature_map_dropout", "hidden_dropout"]
        param_dict = self.load_params(param_list, kwargs)
        self.__dict__.update(param_dict)
        self.hidden_size_2 = self.hidden_size // self.hidden_size_1
        k = self.hidden_size
        self.ent_embeddings = NamedEmbedding("ent_embedding", self.tot_entity, k)
        # reciprocal relations: every relation has a mirrored reverse (projection.py:40-42)
        self.rel_embeddings = NamedEmbedding("rel_embedding", self.tot_relation * 2, k)
        self.b = NamedEmbedding("b", 1, self.tot_entity)
        self.bn0 = nn.BatchNorm2d(1)
        self.inp_drop = nn.Dropout(self.input_dropout)
        self.conv2d_1 = nn.Conv2d(1, 32, (3, 3), stride=(1, 1))
        self.bn1 = nn.BatchNorm2d(32)
        self.feat_drop = nn.Dropout2d(self.feature_map_dropout)
        self.fc = nn.Linear((2 * self.hidden_size_2 - 3 + 1) * (self.hidden_size_1 - 3 + 1) * 32, k)
        self.hidden_drop = nn.Dropout(self.hidden_dropout)
        self.bn2 = nn.BatchNorm1d(k)
        self.parameter_list = [self.ent_embeddings, self.rel_embeddings, self.b]
        self.loss = Criterion.multi_class_bce
        self.kge_trunk = bool(kwargs.get("kge_trunk", True))

    def embed(self, h, r, t):
        return self.ent_embeddings(h), self.rel_embeddings(r), self.ent_embeddings(t)

    def embed2(self, e, r):
        return self.ent_embeddings(e), self.rel_embeddings(r)

    def _kernel_trunk(self):
        """the kernels are selected and the tables live on a CUDA device (the kernels read device memory only)"""
        return self.kge_trunk and self.ent_embeddings.weight.is_cuda

    def kge_train_supported(self):
        """kge_conve_train_* runs this model's training trunk: kernels selected, an image they take (as
        kge_conve_trunk_fwd: hidden_size_1 >= 3, hidden_size_2 >= 2, 2k <= 4096) and BatchNorms with running
        statistics and a momentum"""
        k, h1 = int(self.hidden_size), int(self.hidden_size_1)
        bns = (self.bn0, self.bn1, self.bn2)
        return self._kernel_trunk() and h1 >= 3 and k % h1 == 0 and k // h1 >= 2 and 2 * k <= 4096 and \
            all(bn.track_running_stats and bn.momentum is not None for bn in bns)

    def kge_conve_params(self):
        """the 12 trunk tensors in parameters() order without the bias row b (kge_conve_train_bwd's gradient order)"""
        return [self.ent_embeddings.weight, self.rel_embeddings.weight, self.bn0.weight, self.bn0.bias,
                self.conv2d_1.weight, self.conv2d_1.bias, self.bn1.weight, self.bn1.bias, self.fc.weight,
                self.fc.bias, self.bn2.weight, self.bn2.bias]

    def dropout_noise(self, rows):
        """(noise0 [rows, 2k], noise1 [rows, 32], noise2 [rows, k]) of inp_drop, feat_drop (Dropout2d: one value per
        channel) and hidden_drop in training mode, drawn in that order as ATen draws bernoulli noise: each None when
        its p is 0 or in eval mode, zeros when p >= 1"""
        w = self.ent_embeddings.weight
        out = []
        for drop, width in ((self.inp_drop, 2 * self.hidden_size), (self.feat_drop, 32), (self.hidden_drop,
                                                                                           self.hidden_size)):
            p = float(drop.p)
            if p == 0.0 or not self.training:
                out.append(None)
            elif p >= 1.0:
                out.append(torch.zeros((rows, width), dtype=torch.float32, device=w.device))
            else:
                out.append(torch.empty((rows, width), dtype=torch.float32, device=w.device).bernoulli_(1 - p)
                           .div_(1 - p))
        return tuple(out)

    def note_batch_stats(self, forwards=1):
        """num_batches_tracked += forwards on the three BatchNorms (kge_conve_train_fwd updates the rest)"""
        for bn in (self.bn0, self.bn1, self.bn2):
            bn.num_batches_tracked.add_(forwards)

    def _train_trunk(self, e, r):
        """the training-mode trunk: ConveTrunkFunction where the kernels take it, else the torch layers"""
        B = e.shape[0]
        if B == 0 or not self.kge_train_supported():
            return self._trunk_layers(e, r)
        if B == 1:   # nn.BatchNorm1d's refusal (bn2), before anything runs
            raise ValueError("Expected more than 1 value per channel when training, got input size %s"
                             % (torch.Size([1, int(self.hidden_size)]),))
        x = ConveTrunkFunction.apply(self, e, r, B, *self.dropout_noise(B), *self.kge_conve_params())
        self.note_batch_stats()
        return x

    # ---- trunk: everything of inner_forward before the x . E^T product (projection.py:88-99) ----
    def _trunk_layers(self, e, r):
        e_emb, r_emb = self.embed2(e, r)
        stacked_e = e_emb.view(-1, 1, self.hidden_size_2, self.hidden_size_1)
        stacked_r = r_emb.view(-1, 1, self.hidden_size_2, self.hidden_size_1)
        x = torch.cat([stacked_e, stacked_r], 2)
        x = self.bn0(x)
        x = self.inp_drop(x)
        x = _conv2d_fp32(self.conv2d_1, x)
        x = self.bn1(x)
        x = torch.relu(x)
        x = self.feat_drop(x)
        x = x.view(e.shape[0], -1)
        x = self.fc(x)
        x = self.hidden_drop(x)
        if self.training:
            x = self.bn2(x)   # the reference applies bn2 in training mode only (projection.py:97-98)
        return torch.relu(x)

    def _rel_ids(self, r, direction):
        assert direction in ("head", "tail"), "Unknown forward direction"
        return r + self.tot_relation if direction == "head" else r

    def proj_query(self, e, r, direction="tail"):
        """x [b, k]: the operand of the tail product, for the batched Evaluator (eval mode)."""
        _require_cuda(e, r, self.ent_embeddings.weight)
        r = self._rel_ids(r, direction)
        if not self.training and not torch.is_grad_enabled():
            return _lib.conve_trunk_fwd(self, e.contiguous(), r.contiguous())
        return self._train_trunk(e, r) if self.training else self._trunk_layers(e, r)

    def proj_tail_tables(self):
        """(entity table [N,k], bias row [N]) of the tail product."""
        return self.ent_embeddings.weight, self.b.weight.view(-1)

    def forward(self, e, r, direction="tail"):
        if self.training:
            x = self._train_trunk(e, self._rel_ids(r, direction))
        elif torch.is_grad_enabled():
            x = self._trunk_layers(e, self._rel_ids(r, direction))
        else:
            x = self.proj_query(e, r, direction)
        return ProjTailFunction.apply(x, self.ent_embeddings.weight, self.b.weight)

    def predict_tail_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="tail"), k=topk)
        return rank

    def predict_head_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="head"), k=topk)
        return rank


def _philox_key(device, count):
    """(seed, offset) of `count` counter-mode draws, taken from torch's CUDA generator of `device`: the seed is the
    generator's (torch.manual_seed), the offset its Philox offset, which is advanced past the draws as an ATen
    kernel would, so consecutive calls use disjoint counters and a reseeded run repeats."""
    gen = torch.cuda.default_generators[device.index if device.index is not None else torch.cuda.current_device()]
    seed, offset = gen.initial_seed(), gen.get_offset()
    gen.set_offset(offset + 4 * ((count + 3) // 4))
    return seed, offset


class TuckerTrunkFunction(torch.autograd.Function):
    """x = TuckER's trunk (projection.py:318-328) on kge_tucker_cores -> kge_tucker_trunk_fwd; backward runs
    kge_tucker_trunk_bwd -> kge_tucker_cores_bwd.  One core matrix per distinct relation of the batch is built and
    kept for the backward ([U, d1*d1]); no [B, d1, d1] tensor exists.  mask: None, ("explicit", noise1) or
    ("counter", seed, offset, p)."""

    @staticmethod
    def forward(ctx, e, r, noise0, mask, noise2, ent, rel, W):
        _require_cuda(e, r, ent, rel, W)
        tabs = [ent.detach().contiguous(), rel.detach().contiguous(), W.detach().contiguous()]
        ids, slot = torch.unique(r, return_inverse=True)
        slot = slot.contiguous()
        kw = {}
        if mask is not None:
            kw = {"noise1": mask[1].contiguous()} if mask[0] == "explicit" else {"counter": tuple(mask[1:])}
        kw.update(noise0=noise0, noise2=noise2)
        M = _lib.tucker_cores(tabs, ids)
        x, xpre, nrm = _lib.tucker_trunk_fwd(tabs, M, e.contiguous(), slot, save=True, **kw)
        ctx.kw = kw
        ctx.save_for_backward(e.contiguous(), ids, slot, M, xpre, nrm, *tabs)
        return x

    @staticmethod
    def backward(ctx, gx):
        e, ids, slot, M, xpre, nrm, ent, rel, W = ctx.saved_tensors
        tabs = [ent, rel, W]
        need = ctx.needs_input_grad[5:8]
        gent = torch.zeros_like(ent) if need[0] else None
        dM = torch.zeros_like(M) if (need[1] or need[2]) else None
        _lib.tucker_trunk_bwd(tabs, M, e, slot, gx.contiguous(), xpre, nrm, gent, dM, **ctx.kw)
        grel = torch.zeros_like(rel) if need[1] else None
        gW = torch.zeros_like(W) if need[2] else None
        if dM is not None:
            _lib.tucker_cores_bwd(tabs, ids, dM, grel, gW)
        return None, None, None, None, None, gent, grel, gW


class TuckerCores:
    """The core matrices of a set of relations for evaluation (TuckER.proj_query_cores): built once, reused by every
    query batch and both directions.  At most `budget_bytes` of matrices are held: when the relations need more,
    they are split into chunks of budget_bytes // (4 d1^2) relations and the chunk a batch needs is (re)built on
    demand, one at a time.  A core matrix does not depend on which other relations share its kernel call, so
    chunking never changes x.  The matrices are a snapshot of rel and W: do not keep this object across a weight
    update (the fused optimizer kernels write through raw pointers, which torch's version counters do not see)."""

    def __init__(self, tables, rel_ids, budget_bytes):
        self.tables = [t.detach() for t in tables]
        d1 = self.tables[0].shape[1]
        self.ids = torch.unique(rel_ids)   # sorted
        self.per = max(1, int(budget_bytes) // (4 * d1 * d1))
        self.builds = 0
        self._chunk = (-1, None)
        if self.ids.numel() <= self.per:
            self._cores(0)

    def _cores(self, c):
        if self._chunk[0] != c:
            self._chunk = (-1, None)   # release the held chunk before the next one is allocated
            self._chunk = (c, _lib.tucker_cores(self.tables, self.ids[c * self.per:(c + 1) * self.per].contiguous()))
            self.builds += 1
        return self._chunk[1]

    def query(self, e, r):
        """x [Q, d1] for entity ids e and relation ids r (every r must be among the ids given at construction)"""
        slot = torch.searchsorted(self.ids, r)
        if self.ids.numel() <= self.per:
            return _lib.tucker_trunk_fwd(self.tables, self._cores(0), e, slot)
        x = torch.empty((e.numel(), self.tables[0].shape[1]), dtype=torch.float32, device=e.device)
        chunk = torch.div(slot, self.per, rounding_mode="floor")
        for c in torch.unique(chunk).tolist():
            idx = (chunk == c).nonzero().flatten()
            x[idx] = _lib.tucker_trunk_fwd(self.tables, self._cores(c), e[idx].contiguous(),
                                           (slot[idx] - c * self.per).contiguous())
        return x


class TuckER(ProjectionModel):
    """pykg2vec/models/projection.py:258-345 — same kwargs, tables (ent_embeddings, rel_embeddings, W),
    parameter_list and loss binding.  As in the reference the `direction` argument is validated and otherwise
    ignored: both directions apply the same function, to (h, r) and to (t, r).

    The trunk (normalise, contract the relation with the core tensor, multiply, normalise) runs on the kge_tucker_*
    kernels: one core matrix per distinct relation instead of the reference's one per sample, the dropout on it
    regenerated from a counter.  With autograd (or in training mode) it is TuckerTrunkFunction; in evaluation
    without autograd proj_query takes the matrices from a TuckerCores (proj_query_cores).  The reference's torch
    layers stay as _trunk_layers: the yardstick of the tests, the path for widths the kernels refuse (d1 or
    d2 > 256) and, with the attribute / kwarg kge_trunk = False, for everything."""

    CORES_BUDGET = 256 << 20   # bytes of core matrices a TuckerCores holds at a time

    def __init__(self, **kwargs):
        super(TuckER, self).__init__(self.__class__.__name__.lower())
        param_list = ["tot_entity", "tot_relation", "ent_hidden_size", "rel_hidden_size", "lmbda",
                      "input_dropout", "hidden_dropout1", "hidden_dropout2"]
        param_dict = self.load_params(param_list, kwargs)
        self.__dict__.update(param_dict)
        self.d1, self.d2 = self.ent_hidden_size, self.rel_hidden_size
        self.ent_embeddings = NamedEmbedding("ent_embedding", self.tot_entity, self.d1)
        self.rel_embeddings = NamedEmbedding("rel_embedding", self.tot_relation, self.d2)
        self.W = NamedEmbedding("W", self.d2, self.d1 * self.d1)
        nn.init.xavier_uniform_(self.ent_embeddings.weight)
        nn.init.xavier_uniform_(self.rel_embeddings.weight)
        nn.init.xavier_uniform_(self.W.weight)
        self.parameter_list = [self.ent_embeddings, self.rel_embeddings, self.W]
        self.inp_drop = nn.Dropout(self.input_dropout)
        self.hidden_dropout1 = nn.Dropout(self.hidden_dropout1)
        self.hidden_dropout2 = nn.Dropout(self.hidden_dropout2)
        self.loss = Criterion.multi_class_bce
        self.kge_trunk = bool(kwargs.get("kge_trunk", True))

    def _kernel_trunk(self):
        """the kernels are selected and the tables live on a CUDA device (the kernels read device memory only)"""
        return self.kge_trunk and self.ent_embeddings.weight.is_cuda

    def kge_tucker_tables(self):
        """the three weight tensors in parameter_list order (the C-ABI's kge_tucker_t order)"""
        return [emb.weight for emb in self.parameter_list]

    # ---- trunk: TuckER.forward before the x . E^T product (projection.py:318-328) ----
    def _trunk_layers(self, e1, r):
        e1 = torch.nn.functional.normalize(self.ent_embeddings(e1), p=2, dim=1)
        e1 = self.inp_drop(e1).view(-1, 1, self.d1)
        W_mat = torch.matmul(self.rel_embeddings(r), self.W.weight.view(self.d2, -1)).view(-1, self.d1, self.d1)
        W_mat = self.hidden_dropout1(W_mat)
        x = torch.matmul(e1, W_mat).view(-1, self.d1)
        return self.hidden_dropout2(torch.nn.functional.normalize(x, p=2, dim=1))

    def dropout_noise(self, rows, p):
        """[rows, d1] noise of nn.Dropout(p) in training mode drawn as ATen draws it, or None when nothing drops"""
        p = float(p)
        if p == 0.0 or not self.training:
            return None
        w = self.ent_embeddings.weight
        if p >= 1.0:
            return torch.zeros((rows, self.d1), dtype=torch.float32, device=w.device)
        return torch.empty((rows, self.d1), dtype=torch.float32, device=w.device).bernoulli_(1 - p).div_(1 - p)

    def dropout1_key(self, rows):
        """the counter-mode mask ("counter", seed, offset, p) of hidden_dropout1 over [rows, d1, d1], or None"""
        p = float(self.hidden_dropout1.p)
        if p == 0.0 or not self.training:
            return None
        return ("counter",) + _philox_key(self.ent_embeddings.weight.device, rows * self.d1 * self.d1) + (p,)

    def proj_query_cores(self, rel_ids, budget_bytes=None):
        """The core matrices of the distinct relations in rel_ids (device int64) for proj_query(..., cores=...), or
        None when proj_query would not use them (autograd or training mode, kge_trunk off, unsupported widths).
        Build one per evaluation call, never keep it across a weight update."""
        if self.training or torch.is_grad_enabled() or not self._kernel_trunk():
            return None
        try:
            return TuckerCores(self.kge_tucker_tables(), rel_ids,
                               self.CORES_BUDGET if budget_bytes is None else budget_bytes)
        except _lib.KgeNotSupported:
            return None

    def proj_query(self, e1, r, direction="tail", cores=None):
        assert direction in ("head", "tail"), "Unknown forward direction"
        _require_cuda(e1, r, self.ent_embeddings.weight)
        if not self._kernel_trunk():
            return self._trunk_layers(e1, r)
        e1, r = e1.contiguous(), r.contiguous()
        try:
            if not self.training and not torch.is_grad_enabled():
                cores = cores if cores is not None else self.proj_query_cores(r)
                if cores is None:
                    return self._trunk_layers(e1, r)
                return cores.query(e1, r)
            rows = e1.shape[0]
            return TuckerTrunkFunction.apply(e1, r, self.dropout_noise(rows, self.inp_drop.p), self.dropout1_key(rows),
                                             self.dropout_noise(rows, self.hidden_dropout2.p),
                                             *self.kge_tucker_tables())
        except _lib.KgeNotSupported:   # d1 or d2 beyond the kernels' bound
            return self._trunk_layers(e1, r)

    def proj_tail_tables(self):
        return self.ent_embeddings.weight, None

    def forward(self, e1, r, direction="head"):
        return ProjTailFunction.apply(self.proj_query(e1, r, direction), self.ent_embeddings.weight, None)

    def predict_tail_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="tail"), k=topk)
        return rank

    def predict_head_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="head"), k=topk)
        return rank


def _chequer_perm(hidden_size, reshape_width, P):
    """InteractE's chequer permutation [P, 2*hidden_size] (projection.py:468-505).  numpy draws, in this order,
    P permutations of the entity features, then P of the relation features (np.random.permutation).  Image p
    interleaves them pairwise, entity and relation (offset by hidden_size) features alternating; within every
    run of reshape_width pairs the pair order is (entity, relation) when run index + p is even, else
    (relation, entity)."""
    ent = [np.random.permutation(hidden_size) for _ in range(P)]
    rel = [np.random.permutation(hidden_size) for _ in range(P)]
    run = np.arange(hidden_size) // reshape_width
    rows = []
    for p in range(P):
        e, r = ent[p], rel[p] + hidden_size
        ent_first = ((run + p) % 2 == 0)[:, None]
        rows.append(np.where(ent_first, np.stack([e, r], 1), np.stack([r, e], 1)).reshape(-1))
    return torch.from_numpy(np.stack(rows).astype(np.int64))


class InteracteTrunkFunction(torch.autograd.Function):
    """x = InteractE's trunk in training mode (projection.py:425-442) on kge_interacte_train_fwd; backward runs
    kge_interacte_train_bwd.  The Q = G * B rows are G groups of B rows, each with its own batch statistics; the
    forward updates the model's running statistics in place (num_batches_tracked is the caller's).  noise0 / noise1 /
    noise2: the dropout noise [Q, P*2k] / [Q, P*F] / [Q, k], or None.  params: InteractE.kge_interacte_params().
    The backward reuses the forward's feature-map buffer, so the graph is backpropagated once."""

    @staticmethod
    def forward(ctx, model, e, r, B, noise0, noise1, noise2, *params):
        _require_cuda(e, r, *params)
        params = [t.detach() for t in params]
        e, r = e.contiguous(), r.contiguous()
        perm = model._perm_on(e.device)
        x, ws = _lib.interacte_train_fwd(model, e, r, B, noise0, noise1, noise2, params=params, perm=perm)
        ctx.model, ctx.B, ctx.noise, ctx.perm = model, B, (noise0, noise1, noise2), perm
        ctx.save_for_backward(e, r, x, ws, *params)
        return x

    @staticmethod
    def backward(ctx, gx):
        e, r, x, ws, *params = ctx.saved_tensors
        grads = [torch.zeros_like(t) for t in params]
        _lib.interacte_train_bwd(ctx.model, e, r, ctx.B, gx.contiguous(), x, grads, ws, *ctx.noise, params=params,
                                 perm=ctx.perm)
        return (None,) * 7 + tuple(g if need else None for g, need in zip(grads, ctx.needs_input_grad[7:]))


class InteractE(ProjectionModel):
    """pykg2vec/models/projection.py:347-505 — same kwargs (including the required `device`; hidden_size is read
    and then replaced by reshape_width * reshape_height), sub-module names and state_dict keys (bias / conv_filt /
    ent_embeddings / rel_embeddings / bn0 / bn1 / bn2 / fc), parameter_list and loss binding.  `chequer_perm`
    (int64 [P, 2k]) is drawn from the global np.random at construction with the reference's calls and, as there,
    is a plain attribute: not a parameter or buffer, so not in state_dict.  As in the reference `direction` is
    validated and otherwise ignored: the head direction runs the same function on (t, r).

    In training mode with the tables on a CUDA device the trunk is InteracteTrunkFunction (kge_interacte_train_*);
    the reference's torch layers (the circular convolution through _Fp32Conv2d with TF32 off, so conv_filt trains)
    stay as _trunk_layers: the yardstick of the tests, the path for CPU tables, for geometries the kernels refuse, for
    BatchNorms with momentum None or without running statistics, for a chequer_perm whose rows are not permutations
    of 0 .. 2k-1 and, with the attribute / kwarg kge_trunk = False, for everything.  Evaluation without autograd runs
    kge_interacte_trunk_fwd — one kernel for gather + permutation + bn0 + circular conv + bn1 + ReLU, the Linear
    layer on the tail's tiled GEMM, then bn2 + ReLU."""

    def __init__(self, **kwargs):
        super(InteractE, self).__init__(self.__class__.__name__.lower())
        param_list = ["tot_entity", "tot_relation", "hidden_size", "input_dropout", "hidden_dropout",
                      "feature_map_dropout", "feature_permutation", "num_filters", "kernel_size", "reshape_height",
                      "reshape_width"]
        param_dict = self.load_params(param_list, kwargs)
        self.__dict__.update(param_dict)
        self.hidden_size = self.reshape_width * self.reshape_height
        self.device = kwargs["device"]
        k, P = self.hidden_size, self.feature_permutation
        # construction order = the reference's: it fixes the state_dict order and the torch / numpy draws
        self.ent_embeddings = NamedEmbedding("ent_embeddings", self.tot_entity, k, padding_idx=None)
        self.rel_embeddings = NamedEmbedding("rel_embeddings", self.tot_relation, k, padding_idx=None)
        self.bceloss = nn.BCELoss()
        self.inp_drop = nn.Dropout(self.input_dropout)
        self.hidden_drop = nn.Dropout(self.hidden_dropout)
        self.feature_map_drop = nn.Dropout2d(self.feature_map_dropout)
        self.bn0 = nn.BatchNorm2d(P)
        self.padding = 0
        self.bn1 = nn.BatchNorm2d(self.num_filters * P)
        self.flat_sz = self.reshape_height * 2 * self.reshape_width * self.num_filters * P
        self.bn2 = nn.BatchNorm1d(k)
        self.fc = nn.Linear(self.flat_sz, k)
        self.chequer_perm = _chequer_perm(k, self.reshape_width, P).to(self.device)
        self.register_parameter("bias", nn.Parameter(torch.zeros(self.tot_entity)))
        self.register_parameter("conv_filt", nn.Parameter(torch.zeros(self.num_filters, 1, self.kernel_size,
                                                                      self.kernel_size)))
        nn.init.xavier_uniform_(self.ent_embeddings.weight)
        nn.init.xavier_uniform_(self.rel_embeddings.weight)
        nn.init.xavier_uniform_(self.conv_filt)
        self.parameter_list = [self.ent_embeddings, self.rel_embeddings]
        self.loss = Criterion.multi_class_bce
        self._perm_dev = None
        self._perm_valid = None
        self.kge_trunk = bool(kwargs.get("kge_trunk", True))

    def embed(self, h, r, t):
        return self.ent_embeddings(h), self.rel_embeddings(r), self.ent_embeddings(t)

    def embed2(self, e, r):
        return self.ent_embeddings(e), self.rel_embeddings(r)

    def _perm_on(self, device):
        """chequer_perm as int64 on `device`: copied once per (attribute value, device); the attribute itself stays
        where construction (or the caller) put it"""
        src = self.chequer_perm
        if src.device == device and src.dtype == torch.int64:
            return src
        if self._perm_dev is None or self._perm_dev[0] is not src or self._perm_dev[1].device != device:
            self._perm_dev = (src, src.to(device=device, dtype=torch.int64))
        return self._perm_dev[1]

    def _perm_is_permutation(self):
        """every row of chequer_perm ([P, 2k]) is a permutation of 0 .. 2k-1, which the training kernels' un-permute
        relies on: checked once per attribute value"""
        src = self.chequer_perm
        if self._perm_valid is None or self._perm_valid[0] is not src:
            n, P = 2 * int(self.hidden_size), int(self.feature_permutation)
            ok = tuple(src.shape) == (P, n) and not src.is_floating_point() and not src.is_complex()
            if ok:
                want = torch.arange(n, device=src.device, dtype=torch.int64).expand(P, n)
                ok = bool(torch.equal(torch.sort(src.to(torch.int64), dim=1).values, want))
            self._perm_valid = (src, ok)
        return self._perm_valid[1]

    def _kernel_trunk(self):
        """the kernels are selected and the tables live on a CUDA device (the kernels read device memory only)"""
        return self.kge_trunk and self.ent_embeddings.weight.is_cuda

    def kge_train_supported(self):
        """kge_interacte_train_* runs this model's training trunk: kernels selected, a geometry they take (as
        kge_interacte_trunk_fwd), BatchNorms with running statistics and a momentum, and a chequer_perm whose rows
        are permutations"""
        bns = (self.bn0, self.bn1, self.bn2)
        return self._kernel_trunk() and all(bn.track_running_stats and bn.momentum is not None for bn in bns) and \
            _lib.interacte_train_workspace_bytes(self, 2, 2) > 0 and self._perm_is_permutation()

    def kge_interacte_params(self):
        """the 11 trunk tensors in kge_interacte_train_bwd's gradient order (parameters() without the bias row)"""
        return [self.ent_embeddings.weight, self.rel_embeddings.weight, self.bn0.weight, self.bn0.bias, self.conv_filt,
                self.bn1.weight, self.bn1.bias, self.fc.weight, self.fc.bias, self.bn2.weight, self.bn2.bias]

    def dropout_noise(self, rows):
        """(noise0 [rows, P*2k], noise1 [rows, P*F], noise2 [rows, k]) of inp_drop (on the [rows, P, H, W] images),
        feature_map_drop (Dropout2d: one value per channel) and hidden_drop in training mode, drawn in that order as
        ATen draws bernoulli noise: each None when its p is 0 or in eval mode, zeros when p >= 1"""
        w = self.ent_embeddings.weight
        k, P = int(self.hidden_size), int(self.feature_permutation)
        out = []
        for drop, width in ((self.inp_drop, P * 2 * k), (self.feature_map_drop, P * int(self.num_filters)),
                            (self.hidden_drop, k)):
            p = float(drop.p)
            if p == 0.0 or not self.training:
                out.append(None)
            elif p >= 1.0:
                out.append(torch.zeros((rows, width), dtype=torch.float32, device=w.device))
            else:
                out.append(torch.empty((rows, width), dtype=torch.float32, device=w.device).bernoulli_(1 - p)
                           .div_(1 - p))
        return tuple(out)

    def note_batch_stats(self, forwards=1):
        """num_batches_tracked += forwards on the three BatchNorms (kge_interacte_train_fwd updates the rest)"""
        for bn in (self.bn0, self.bn1, self.bn2):
            bn.num_batches_tracked.add_(forwards)

    def _train_trunk(self, e, r):
        """the training-mode trunk: InteracteTrunkFunction where the kernels take it, else the torch layers"""
        B = e.shape[0]
        if B == 0 or not self.kge_train_supported():
            return self._trunk_layers(e, r)
        if B == 1:   # nn.BatchNorm1d's refusal (bn2), before anything runs
            raise ValueError("Expected more than 1 value per channel when training, got input size %s"
                             % (torch.Size([1, int(self.hidden_size)]),))
        x = InteracteTrunkFunction.apply(self, e, r, B, *self.dropout_noise(B), *self.kge_interacte_params())
        self.note_batch_stats()
        return x

    # ---- trunk: InteractE.forward before the x . E^T product (projection.py:427-442) ----
    def _trunk_layers(self, e, r):
        e_emb, r_emb = self.embed2(e, r)
        comb = torch.cat([e_emb, r_emb], dim=-1)
        H, W, P = 2 * self.reshape_width, self.reshape_height, self.feature_permutation
        x = comb[:, self._perm_on(comb.device)].reshape(-1, P, H, W)
        x = self.bn0(x)
        x = self.inp_drop(x)
        pad = self.kernel_size // 2
        x = torch.cat([x[..., H - pad:, :], x, x[..., :pad, :]], dim=2)     # circular padding, rows then columns
        x = torch.cat([x[..., W - pad:], x, x[..., :pad]], dim=3)
        # filter f on every image: output channel p*F + f (TF32 off, see _Fp32Conv2d)
        x = _Fp32Conv2d.apply(x, self.conv_filt.repeat(P, 1, 1, 1), None, (1, 1), (self.padding, self.padding),
                              (1, 1), P)
        x = self.bn1(x)
        x = torch.relu(x)
        x = self.feature_map_drop(x)
        x = x.view(-1, self.flat_sz)
        x = self.fc(x)
        x = self.hidden_drop(x)
        x = self.bn2(x)
        return torch.relu(x)

    def proj_query(self, e, r, direction="tail"):
        """x [b, k]: the operand of the tail product, for the batched Evaluator (eval mode)."""
        assert direction in ("head", "tail"), "Unknown forward direction"
        _require_cuda(e, r, self.ent_embeddings.weight)
        if not self.training and not torch.is_grad_enabled():
            return _lib.interacte_trunk_fwd(self, e.contiguous(), r.contiguous(), perm=self._perm_on(e.device))
        return self._train_trunk(e, r) if self.training else self._trunk_layers(e, r)

    def proj_tail_tables(self):
        """(entity table [N,k], bias row [N]) of the tail product."""
        return self.ent_embeddings.weight, self.bias

    def forward(self, e, r, direction="tail"):
        return ProjTailFunction.apply(self.proj_query(e, r, direction), self.ent_embeddings.weight, self.bias)

    def predict_tail_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="tail"), k=topk)
        return rank

    def predict_head_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="head"), k=topk)
        return rank


class HyperTrunkFunction(torch.autograd.Function):
    """x = HypER's trunk in training mode (projection.py:581-606) on kge_hyper_train_fwd; backward runs
    kge_hyper_train_bwd.  The Q = G * B rows are G groups of B rows, each with its own batch statistics; the forward
    updates the model's running statistics in place (num_batches_tracked is the caller's).  noise0 / noise1 / noise2:
    the dropout noise [Q, de] / [Q, 32] / [Q, de], or None.  params: HypER.kge_hyper_params()."""

    @staticmethod
    def forward(ctx, model, e, r, B, noise0, noise1, noise2, *params):
        _require_cuda(e, r, *params)
        params = [t.detach() for t in params]
        e, r = e.contiguous(), r.contiguous()
        x, ws = _lib.hyper_train_fwd(model, e, r, B, noise0, noise1, noise2, params=params)
        ctx.model, ctx.B, ctx.noise = model, B, (noise0, noise1, noise2)
        ctx.save_for_backward(e, r, x, ws, *params)
        return x

    @staticmethod
    def backward(ctx, gx):
        e, r, x, ws, *params = ctx.saved_tensors
        grads = [torch.zeros_like(t) for t in params]
        _lib.hyper_train_bwd(ctx.model, e, r, ctx.B, gx.contiguous(), x, grads, ws, *ctx.noise, params=params)
        return (None,) * 7 + tuple(g if need else None for g, need in zip(grads, ctx.needs_input_grad[7:]))


class HypER(ProjectionModel):
    """pykg2vec/models/projection.py:508-618 — same kwargs (including the required `device`), sub-module
    names (state_dict keys b / ent_embeddings / rel_embeddings / bn0 / bn1 / bn2 / fc / fc1, padding_idx=0 on
    both embeddings), parameter_list and loss binding.  As in the reference `direction` is validated and
    otherwise ignored: the head direction runs the same function on (t, r).

    In training mode with the tables on a CUDA device the trunk is HyperTrunkFunction (kge_hyper_train_*); the
    reference's torch layers stay as _trunk_layers: the yardstick of the tests, the path for CPU tables, for widths
    the kernels refuse (de < 9 or de > 4096), for BatchNorms with momentum None or without running statistics and,
    with the attribute / kwarg kge_trunk = False, for everything."""

    def __init__(self, **kwargs):
        super(HypER, self).__init__(self.__class__.__name__.lower())
        param_list = ["tot_entity", "tot_relation", "ent_hidden_size", "rel_hidden_size", "input_dropout",
                      "hidden_dropout", "feature_map_dropout"]
        param_dict = self.load_params(param_list, kwargs)
        self.__dict__.update(param_dict)
        self.device = kwargs["device"]
        self.filt_h, self.filt_w = 1, 9
        self.in_channels, self.out_channels = 1, 32
        de, dr = self.ent_hidden_size, self.rel_hidden_size
        self.ent_embeddings = NamedEmbedding("ent_embeddings", self.tot_entity, de, padding_idx=0)
        self.rel_embeddings = NamedEmbedding("rel_embeddings", self.tot_relation, dr, padding_idx=0)
        self.inp_drop = nn.Dropout(self.input_dropout)
        self.hidden_drop = nn.Dropout(self.hidden_dropout)
        self.feature_map_drop = nn.Dropout2d(self.feature_map_dropout)
        self.bn0 = nn.BatchNorm2d(self.in_channels)
        self.bn1 = nn.BatchNorm2d(self.out_channels)
        self.bn2 = nn.BatchNorm1d(de)
        self.register_parameter("b", nn.Parameter(torch.zeros(self.tot_entity)))
        self.fc = nn.Linear((1 - self.filt_h + 1) * (de - self.filt_w + 1) * self.out_channels, de)
        self.fc1 = nn.Linear(dr, self.in_channels * self.out_channels * self.filt_h * self.filt_w)
        nn.init.xavier_uniform_(self.ent_embeddings.weight.data)
        nn.init.xavier_uniform_(self.rel_embeddings.weight.data)
        self.parameter_list = [self.ent_embeddings, self.rel_embeddings]
        self.loss = Criterion.multi_class_bce
        self.kge_trunk = bool(kwargs.get("kge_trunk", True))

    def embed(self, h, r, t):
        return self.ent_embeddings(h), self.rel_embeddings(r), self.ent_embeddings(t)

    def embed2(self, e, r):
        return self.ent_embeddings(e), self.rel_embeddings(r)

    def _kernel_trunk(self):
        """the kernels are selected and the tables live on a CUDA device (the kernels read device memory only)"""
        return self.kge_trunk and self.ent_embeddings.weight.is_cuda

    def kge_train_supported(self):
        """kge_hyper_train_* runs this model's training trunk: kernels selected, a width they take (as
        kge_hyper_trunk_fwd: 9 <= de <= 4096) and BatchNorms with running statistics and a momentum"""
        bns = (self.bn0, self.bn1, self.bn2)
        return self._kernel_trunk() and 9 <= int(self.ent_hidden_size) <= 4096 and \
            all(bn.track_running_stats and bn.momentum is not None for bn in bns)

    def kge_hyper_params(self):
        """the 12 trunk tensors in kge_hyper_train_bwd's gradient order (parameters() without the bias row b, bn2
        after fc)"""
        return [self.ent_embeddings.weight, self.rel_embeddings.weight, self.bn0.weight, self.bn0.bias,
                self.bn1.weight, self.bn1.bias, self.fc.weight, self.fc.bias, self.bn2.weight, self.bn2.bias,
                self.fc1.weight, self.fc1.bias]

    def dropout_noise(self, rows):
        """(noise0 [rows, de], noise1 [rows, 32], noise2 [rows, de]) of inp_drop, feature_map_drop (Dropout2d: one
        value per channel) and hidden_drop in training mode, drawn in that order as ATen draws bernoulli noise: each
        None when its p is 0 or in eval mode, zeros when p >= 1"""
        w = self.ent_embeddings.weight
        de = int(self.ent_hidden_size)
        out = []
        for drop, width in ((self.inp_drop, de), (self.feature_map_drop, self.out_channels), (self.hidden_drop, de)):
            p = float(drop.p)
            if p == 0.0 or not self.training:
                out.append(None)
            elif p >= 1.0:
                out.append(torch.zeros((rows, width), dtype=torch.float32, device=w.device))
            else:
                out.append(torch.empty((rows, width), dtype=torch.float32, device=w.device).bernoulli_(1 - p)
                           .div_(1 - p))
        return tuple(out)

    def note_batch_stats(self, forwards=1):
        """num_batches_tracked += forwards on the three BatchNorms (kge_hyper_train_fwd updates the rest)"""
        for bn in (self.bn0, self.bn1, self.bn2):
            bn.num_batches_tracked.add_(forwards)

    def _train_trunk(self, e, r):
        """the training-mode trunk: HyperTrunkFunction where the kernels take it, else the torch layers"""
        B = e.shape[0]
        if B == 0 or not self.kge_train_supported():
            return self._trunk_layers(e, r)
        if B == 1:   # nn.BatchNorm1d's refusal (bn2), before anything runs
            raise ValueError("Expected more than 1 value per channel when training, got input size %s"
                             % (torch.Size([1, int(self.ent_hidden_size)]),))
        x = HyperTrunkFunction.apply(self, e, r, B, *self.dropout_noise(B), *self.kge_hyper_params())
        self.note_batch_stats()
        return x

    # ---- trunk: HypER.forward before the x . E^T product (projection.py:583-606) ----
    def _trunk_layers(self, e, r):
        e_emb, r_emb = self.embed2(e, r)
        B, de = e_emb.size(0), self.ent_embeddings.weight.size(1)
        x = self.bn0(e_emb.view(-1, 1, 1, de))
        x = self.inp_drop(x)
        k = self.fc1(r_emb)
        k = k.view(-1, self.in_channels, self.out_channels, self.filt_h, self.filt_w)
        k = k.view(B * self.in_channels * self.out_channels, 1, self.filt_h, self.filt_w)
        x = x.permute(1, 0, 2, 3)
        # one group per query: query i's 32 filters see only its own row (TF32 off, see _Fp32Conv2d)
        x = _Fp32Conv2d.apply(x, k, None, (1, 1), (0, 0), (1, 1), B)
        x = x.view(B, 1, self.out_channels, 1 - self.filt_h + 1, de - self.filt_w + 1)
        x = x.permute(0, 3, 4, 1, 2)
        x = torch.sum(x, dim=3)
        x = x.permute(0, 3, 1, 2).contiguous()
        x = self.bn1(x)
        x = self.feature_map_drop(x)
        x = x.view(B, -1)
        x = self.fc(x)
        x = self.hidden_drop(x)
        x = self.bn2(x)   # applied in both modes (unlike ConvE)
        return torch.relu(x)

    def proj_query(self, e, r, direction="tail"):
        """x [b, de]: the operand of the tail product, for the batched Evaluator (eval mode)."""
        assert direction in ("head", "tail"), "Unknown forward direction"
        _require_cuda(e, r, self.ent_embeddings.weight)
        if not self.training and not torch.is_grad_enabled():
            return _lib.hyper_trunk_fwd(self, e.contiguous(), r.contiguous())
        return self._train_trunk(e, r) if self.training else self._trunk_layers(e, r)

    def proj_tail_tables(self):
        """(entity table [N,de], bias row [N]) of the tail product."""
        return self.ent_embeddings.weight, self.b

    def forward(self, e, r, direction="tail"):
        return ProjTailFunction.apply(self.proj_query(e, r, direction), self.ent_embeddings.weight, self.b)

    def predict_tail_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="tail"), k=topk)
        return rank

    def predict_head_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="head"), k=topk)
        return rank


class AcreTrunkFunction(torch.autograd.Function):
    """x = AcrE's trunk in training mode (projection.py:706-734) on kge_acre_train_fwd; backward runs
    kge_acre_train_bwd.  The Q = G * B rows are G groups of B rows, each with its own batch statistics; the forward
    updates the model's running statistics in place (num_batches_tracked is the caller's).  noise0 / noise1 / noise2:
    the dropout noise [Q, 400] / [Q, C] / [Q, 200], or None.  params: AcrE.kge_acre_params().  The backward reuses the
    forward's feature buffers, so the graph is backpropagated once."""

    @staticmethod
    def forward(ctx, model, e, r, B, noise0, noise1, noise2, *params):
        _require_cuda(e, r, *params)
        params = [t.detach() for t in params]
        e, r = e.contiguous(), r.contiguous()
        x, ws = _lib.acre_train_fwd(model, e, r, B, noise0, noise1, noise2, params=params)
        ctx.model, ctx.B, ctx.noise = model, B, (noise0, noise1, noise2)
        ctx.save_for_backward(e, r, x, ws, *params)
        return x

    @staticmethod
    def backward(ctx, gx):
        e, r, x, ws, *params = ctx.saved_tensors
        grads = [torch.zeros_like(t) for t in params]
        _lib.acre_train_bwd(ctx.model, e, r, ctx.B, gx.contiguous(), x, grads, ws, *ctx.noise, params=params)
        return (None,) * 7 + tuple(g if need else None for g, need in zip(grads, ctx.needs_input_grad[7:]))


class AcrE(ProjectionModel):
    """pykg2vec/models/projection.py:621-746 — same kwargs, sub-module names and state_dict keys and order (bias /
    ent_embeddings / rel_embeddings / bn0 / bn1 / bn2 / fc / conv1 / conv2 / conv3, then W_gate_e in the parallel
    way), parameter_list and loss binding.  rel_embeddings has 2 * tot_relation rows, but as in the reference
    `direction` is validated and otherwise ignored: both directions index it with r as given (rows R..2R-1 are
    never read) and the head direction runs the same function on (t, r).  The trunk views each 200-wide row as
    10 x 20, so hidden_size must be 200 for the reference's forward to mean anything; the class constructs for
    any size, as upstream, and the evaluation kernel refuses the others (KgeNotSupported).

    In training mode with the tables on a CUDA device the trunk is AcreTrunkFunction (kge_acre_train_*); the
    reference's torch layers (the three convolutions through _Fp32Conv2d with their dilation and padding, TF32 off)
    stay as _trunk_layers: the yardstick of the tests, the path for CPU tables, for configurations the kernels refuse
    (hidden_size != 200, where the reference's own view error surfaces, or more channels than they take), for
    BatchNorms with momentum None or without running statistics and, with the attribute / kwarg kge_trunk = False,
    for everything.  Evaluation without autograd runs kge_acre_trunk_fwd."""

    def __init__(self, **kwargs):
        super(AcrE, self).__init__(self.__class__.__name__.lower())
        param_list = ["tot_entity", "tot_relation", "hidden_size", "input_dropout", "hidden_dropout",
                      "feature_map_dropout", "in_channels", "way", "first_atrous", "second_atrous", "third_atrous",
                      "acre_bias"]
        param_dict = self.load_params(param_list, kwargs)
        self.__dict__.update(param_dict)
        k, C = self.hidden_size, self.in_channels
        # construction order = the reference's: it fixes the state_dict order and the torch draws
        self.ent_embeddings = NamedEmbedding("ent_embedding", self.tot_entity, k, padding_idx=None)
        self.rel_embeddings = NamedEmbedding("rel_embedding", self.tot_relation * 2, k, padding_idx=None)
        self.inp_drop = nn.Dropout(self.input_dropout)
        self.hidden_drop = nn.Dropout(self.hidden_dropout)
        self.feature_map_drop = nn.Dropout2d(self.feature_map_dropout)
        self.bn0 = nn.BatchNorm2d(1)
        self.bn1 = nn.BatchNorm2d(C)
        self.bn2 = nn.BatchNorm1d(k)
        self.fc = nn.Linear(C * 400, k)
        self.padding = 0
        # conv l: 3x3, stride 1, padding = dilation = its atrous rate; serial: 1 -> C -> C -> C, else three 1 -> C
        cin = C if self.way == "serial" else 1
        self.conv1 = nn.Conv2d(1, C, (3, 3), 1, self.first_atrous, bias=self.acre_bias, dilation=self.first_atrous)
        self.conv2 = nn.Conv2d(cin, C, (3, 3), 1, self.second_atrous, bias=self.acre_bias,
                               dilation=self.second_atrous)
        self.conv3 = nn.Conv2d(cin, C, (3, 3), 1, self.third_atrous, bias=self.acre_bias, dilation=self.third_atrous)
        if self.way != "serial":
            self.W_gate_e = nn.Linear(1600, 400)
        self.register_parameter("bias", nn.Parameter(torch.zeros(self.tot_entity)))
        nn.init.xavier_uniform_(self.ent_embeddings.weight.data)
        nn.init.xavier_uniform_(self.rel_embeddings.weight.data)
        self.parameter_list = [self.ent_embeddings, self.rel_embeddings]
        self.loss = Criterion.multi_class_bce
        self.kge_trunk = bool(kwargs.get("kge_trunk", True))

    def embed(self, h, r, t):
        return self.ent_embeddings(h), self.rel_embeddings(r), self.ent_embeddings(t)

    def embed2(self, e, r):
        return self.ent_embeddings(e), self.rel_embeddings(r)

    def _kernel_trunk(self):
        """the kernels are selected and the tables live on a CUDA device (the kernels read device memory only)"""
        return self.kge_trunk and self.ent_embeddings.weight.is_cuda

    def kge_train_supported(self):
        """kge_acre_train_* runs this model's training trunk: kernels selected, a configuration they take
        (hidden_size 200; serial in_channels <= 46, parallel <= 1024) and BatchNorms with running statistics and a
        momentum"""
        bns = (self.bn0, self.bn1, self.bn2)
        return self._kernel_trunk() and all(bn.track_running_stats and bn.momentum is not None for bn in bns) and \
            self._kge_train_config_ok()

    def _kge_train_config_ok(self):
        """kge_acre_train_workspace_bytes accepts this configuration: asked once per configuration, not per step"""
        key = (self.way, int(self.in_channels), int(self.ent_embeddings.weight.shape[1]),
               int(self.rel_embeddings.weight.shape[0]), int(self.first_atrous), int(self.second_atrous),
               int(self.third_atrous))
        if getattr(self, "_kge_train_ok", (None,))[0] != key:
            self._kge_train_ok = (key, _lib.acre_train_workspace_bytes(self, 2, 2) > 0)
        return self._kge_train_ok[1]

    def kge_acre_params(self):
        """the trunk tensors this model has, in kge_acre_train_bwd's slot order (parameters() without the bias row):
        ent, rel, bn0.*, conv1.*, conv2.*, conv3.* (biases with acre_bias only), W_gate_e.* (parallel way only),
        bn1.*, fc.*, bn2.*"""
        out = [self.ent_embeddings.weight, self.rel_embeddings.weight, self.bn0.weight, self.bn0.bias]
        for conv in (self.conv1, self.conv2, self.conv3):
            out += [conv.weight] + ([conv.bias] if conv.bias is not None else [])
        if self.way != "serial":
            out += [self.W_gate_e.weight, self.W_gate_e.bias]
        return out + [self.bn1.weight, self.bn1.bias, self.fc.weight, self.fc.bias, self.bn2.weight, self.bn2.bias]

    def dropout_noise(self, rows):
        """(noise0 [rows, 400], noise1 [rows, C], noise2 [rows, 200]) of inp_drop (on the [rows, 1, 20, 20] image),
        feature_map_drop (Dropout2d: one value per channel) and hidden_drop in training mode, drawn in that order as
        ATen draws bernoulli noise: each None when its p is 0 or in eval mode, zeros when p >= 1"""
        w = self.ent_embeddings.weight
        out = []
        for drop, width in ((self.inp_drop, 400), (self.feature_map_drop, int(self.in_channels)),
                            (self.hidden_drop, int(self.hidden_size))):
            p = float(drop.p)
            if p == 0.0 or not self.training:
                out.append(None)
            elif p >= 1.0:
                out.append(torch.zeros((rows, width), dtype=torch.float32, device=w.device))
            else:
                out.append(torch.empty((rows, width), dtype=torch.float32, device=w.device).bernoulli_(1 - p)
                           .div_(1 - p))
        return tuple(out)

    def note_batch_stats(self, forwards=1):
        """num_batches_tracked += forwards on the three BatchNorms (kge_acre_train_fwd updates the rest)"""
        for bn in (self.bn0, self.bn1, self.bn2):
            bn.num_batches_tracked.add_(forwards)

    def _train_trunk(self, e, r):
        """the training-mode trunk: AcreTrunkFunction where the kernels take it, else the torch layers"""
        B = e.shape[0]
        if B == 0 or not self.kge_train_supported():
            return self._trunk_layers(e, r)
        if B == 1:   # nn.BatchNorm1d's refusal (bn2), before anything runs
            raise ValueError("Expected more than 1 value per channel when training, got input size %s"
                             % (torch.Size([1, int(self.hidden_size)]),))
        x = AcreTrunkFunction.apply(self, e, r, B, *self.dropout_noise(B), *self.kge_acre_params())
        self.note_batch_stats()
        return x

    # ---- trunk: AcrE.forward before the x . E^T product (projection.py:708-734) ----
    def _trunk_layers(self, e, r):
        emb_e, emb_r = self.embed2(e, r)
        x = torch.cat([emb_e.view(-1, 1, 10, 20), emb_r.view(-1, 1, 10, 20)], dim=2)
        x = self.bn0(x)
        x = self.inp_drop(x)
        res = x
        C = self.in_channels
        if self.way == "serial":
            x = _conv2d_fp32(self.conv1, x)
            x = _conv2d_fp32(self.conv2, x)
            x = _conv2d_fp32(self.conv3, x)
            x = x + res
        else:
            conv1 = _conv2d_fp32(self.conv1, x).view(-1, C, 400)
            conv2 = _conv2d_fp32(self.conv2, x).view(-1, C, 400)
            conv3 = _conv2d_fp32(self.conv3, x).view(-1, C, 400)
            res = res.expand(-1, C, 20, 20).view(-1, C, 400)
            x = torch.cat((res, conv1, conv2, conv3), dim=2)
            x = self.W_gate_e(x).view(-1, C, 20, 20)
        x = self.bn1(x)
        x = torch.relu(x)
        x = self.feature_map_drop(x)
        x = x.view(x.shape[0], -1)
        x = self.fc(x)
        x = self.hidden_drop(x)
        x = self.bn2(x)   # applied in both modes (unlike ConvE)
        return torch.relu(x)

    def proj_query(self, e, r, direction="tail"):
        """x [b, k]: the operand of the tail product, for the batched Evaluator (eval mode)."""
        assert direction in ("head", "tail"), "Unknown forward direction"
        _require_cuda(e, r, self.ent_embeddings.weight)
        if not self.training and not torch.is_grad_enabled():
            return _lib.acre_trunk_fwd(self, e.contiguous(), r.contiguous())
        return self._train_trunk(e, r) if self.training else self._trunk_layers(e, r)

    def proj_tail_tables(self):
        """(entity table [N,k], bias row [N]) of the tail product."""
        return self.ent_embeddings.weight, self.bias

    def forward(self, e, r, direction="tail"):
        return ProjTailFunction.apply(self.proj_query(e, r, direction), self.ent_embeddings.weight, self.bias)

    def predict_tail_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="tail"), k=topk)
        return rank

    def predict_head_rank(self, e, r, topk=-1):
        _, rank = torch.topk(-self.forward(e, r, direction="head"), k=topk)
        return rank


class ProjEFunction(torch.autograd.Function):
    """One direction of ProjE_pointwise.forward (projection.py:194-210): the scalar loss term.  Forward and
    backward both run in kge_proje_train_step during forward(); backward() scales the stored gradients."""

    @staticmethod
    def forward(ctx, direction, e, r, labels, noise, *tables):
        _require_cuda(e, r, labels, *tables)
        tabs = [t.detach() for t in tables]
        grads = [torch.zeros_like(t) if ctx.needs_input_grad[5 + i] else None for i, t in enumerate(tabs)]
        tail = direction == "tail"
        e, r = e.contiguous(), r.contiguous()
        labels = labels.detach().to(torch.float32).contiguous()
        noise = noise.contiguous() if noise is not None else None
        if tail:
            loss = _lib.proje_train_step(tabs, e, r, None, labels, None, grads, noise_tail=noise)
        else:
            loss = _lib.proje_train_step(tabs, None, r, e, None, labels, grads, noise_head=noise)
        ctx.mask = [g is not None for g in grads]
        ctx.save_for_backward(*[g for g in grads if g is not None])
        return loss.squeeze_(0)

    @staticmethod
    def backward(ctx, gout):
        saved = iter(ctx.saved_tensors)
        grads = [next(saved) * gout if m else None for m in ctx.mask]
        return (None, None, None, None, None, *grads)


class L1RegFunction(torch.autograd.Function):
    """lmbda * sum |w| over whole tensors (ProjE_pointwise.get_reg, projection.py:189-192) via kge_reg_l1_dense."""

    @staticmethod
    def forward(ctx, lmbda, *tensors):
        _require_cuda(*tensors)
        ts = [t.detach() for t in tensors]
        grads = [torch.zeros_like(t) if ctx.needs_input_grad[1 + i] else None for i, t in enumerate(ts)]
        out = _lib.reg_l1_dense(ts, grads, float(lmbda))
        ctx.mask = [g is not None for g in grads]
        ctx.save_for_backward(*[g for g in grads if g is not None])
        return out.squeeze_(0)

    @staticmethod
    def backward(ctx, gout):
        saved = iter(ctx.saved_tensors)
        return (None, *[next(saved) * gout if m else None for m in ctx.mask])


class ProjE_pointwise(ProjectionModel):
    """pykg2vec/models/projection.py:128-257 — same kwargs (including the required `device`), the eight
    NamedEmbedding tables with the reference's names and state_dict keys, xavier_uniform_ in the reference's order
    (a seeded construction draws the reference's initial weights), parameter_list, loss binding
    (Criterion.multi_class), f1 / f2 / g and get_reg.

    forward(e, r, er_e2, direction) returns the direction's loss term, as the reference does, through
    ProjEFunction: the hidden dropout (torch.dropout(train=True) on every call, :201-203) is drawn with torch as
    ATen draws it, noise = bernoulli(1 - p) / (1 - p), and multiplied in by the kernel.  The head direction is
    f2(t, r) with plain r (no reciprocal relation).  get_reg is an L1 sum over the whole tables
    (kge_reg_l1_dense).  proj_query / proj_tail_tables feed the batched Evaluator (eval: no dropout, as
    predict_*_rank)."""

    def __init__(self, **kwargs):
        super(ProjE_pointwise, self).__init__(self.__class__.__name__.lower())
        param_list = ["tot_entity", "tot_relation", "hidden_size", "lmbda", "hidden_dropout"]
        param_dict = self.load_params(param_list, kwargs)
        self.__dict__.update(param_dict)
        k = self.hidden_size
        self.device = kwargs["device"]
        self.ent_embeddings = NamedEmbedding("ent_embedding", self.tot_entity, k)
        self.rel_embeddings = NamedEmbedding("rel_embedding", self.tot_relation, k)
        self.bc1 = NamedEmbedding("bc1", 1, k)
        self.De1 = NamedEmbedding("De1", 1, k)
        self.Dr1 = NamedEmbedding("Dr1", 1, k)
        self.bc2 = NamedEmbedding("bc2", 1, k)
        self.De2 = NamedEmbedding("De2", 1, k)
        self.Dr2 = NamedEmbedding("Dr2", 1, k)
        self.parameter_list = [self.ent_embeddings, self.rel_embeddings, self.bc1, self.De1, self.Dr1, self.bc2,
                               self.De2, self.Dr2]
        for emb in self.parameter_list:   # the reference's order: it fixes the torch draws
            nn.init.xavier_uniform_(emb.weight)
        self.loss = Criterion.multi_class

    def kge_proje_tables(self):
        """the eight weight tensors in parameter_list order (the C-ABI's kge_proje_t / gradient order)"""
        return [emb.weight for emb in self.parameter_list]

    def kge_reg_tables(self):
        """(indices into kge_proje_tables(), tensors) of get_reg's L1 sum: De1, Dr1, De2, Dr2, ent, rel"""
        idx = (3, 4, 6, 7, 0, 1)
        tabs = self.kge_proje_tables()
        return idx, [tabs[i] for i in idx]

    def get_reg(self, h, r, t):
        return L1RegFunction.apply(float(self.lmbda), *self.kge_reg_tables()[1])

    def dropout_noise(self, rows):
        """[rows, k] noise of torch.dropout(p=hidden_dropout, train=True) drawn as ATen draws it, or None for p = 0"""
        p = float(self.hidden_dropout)
        if p == 0.0:
            return None
        w = self.ent_embeddings.weight
        if p >= 1.0:
            return torch.zeros((rows, self.hidden_size), dtype=torch.float32, device=w.device)
        return torch.empty((rows, self.hidden_size), dtype=torch.float32, device=w.device).bernoulli_(1 - p).div_(1 - p)

    def forward(self, e, r, er_e2, direction="tail"):
        assert direction in ("head", "tail"), "Unknown forward direction"
        _require_cuda(e, r, self.ent_embeddings.weight)
        return ProjEFunction.apply(direction, e, r, er_e2, self.dropout_noise(e.shape[0]), *self.kge_proje_tables())

    def f1(self, h, r):
        """tanh(h * De1 + r * Dr1 + bc1) of embedding rows (projection.py:212-219)"""
        return torch.tanh(h * self.De1.weight + r * self.Dr1.weight + self.bc1.weight)

    def f2(self, t, r):
        """tanh(t * De2 + r * Dr2 + bc2) of embedding rows (projection.py:221-228)"""
        return torch.tanh(t * self.De2.weight + r * self.Dr2.weight + self.bc2.weight)

    @staticmethod
    def g(f, w):
        """sigmoid(f . w^T) (projection.py:248-257), on kge_proj_tail_fwd"""
        return ProjTailFunction.apply(f, w, None)

    def proj_query(self, e, r, direction="tail"):
        """x [b, k] = f1(e, r) (tail) or f2(e, r) (head) by kge_proje_trunk_fwd, for the batched Evaluator and
        predict_*_rank (no dropout; not differentiable)."""
        assert direction in ("head", "tail"), "Unknown forward direction"
        _require_cuda(e, r, self.ent_embeddings.weight)
        return _lib.proje_trunk_fwd(self.kge_proje_tables(), e.contiguous(), r.contiguous(),
                                    0 if direction == "tail" else 1)

    def proj_tail_tables(self):
        """(entity table [N,k], no bias row) of g()"""
        return self.ent_embeddings.weight, None

    def predict_tail_rank(self, h, r, topk=-1):
        preds = _lib.proj_tail_fwd(self.proj_query(h, r, "tail"), self.ent_embeddings.weight.detach())
        _, rank = torch.topk(-preds, k=topk)
        return rank

    def predict_head_rank(self, t, r, topk=-1):
        preds = _lib.proj_tail_fwd(self.proj_query(t, r, "head"), self.ent_embeddings.weight.detach())
        _, rank = torch.topk(-preds, k=topk)
        return rank
