"""torch.autograd.Function wrappers around the C-ABI kernels.

These are what make the CUDA path a drop-in behind `loss.backward()` of the
reference's Trainer (pykg2vec/utils/trainer.py:298): forward() returns an fp32 [b]
tensor whose backward scatters DENSE gradients into the nn.Embedding weights, exactly
the autograd contract of the reference models.  No CPU / eager fallback exists: CPU
tensors raise.
"""
import torch

from . import _lib


def _require_cuda(*tensors):
    for t in tensors:
        if not t.is_cuda:
            raise _lib.KgeError(
                "pykg2vec_b200 runs on CUDA (sm_90a) only: got a %s tensor. There is no CPU "
                "fallback — move the model and ids to a CUDA device." % t.device)


class ScoreFunction(torch.autograd.Function):
    """model.forward(h, r, t) -> scores [b].  `spec` is the model's static description
    (name, dim, ...), tables are passed explicitly so autograd tracks them."""

    @staticmethod
    def forward(ctx, spec, h, r, t, *tables):
        _require_cuda(h, r, t, *tables)
        h, r, t = h.contiguous(), r.contiguous(), t.contiguous()
        desc = spec.desc([tb.detach() for tb in tables])
        out = _lib.score_fwd(desc, h, r, t, _lib.GROUP_TAIL)
        ctx.spec = spec
        ctx.save_for_backward(h, r, t, *tables)
        return out

    @staticmethod
    def backward(ctx, gout):
        h, r, t, *tables = ctx.saved_tensors
        desc = ctx.spec.desc([tb.detach() for tb in tables])
        grads = []
        for k, tb in enumerate(tables):
            need = ctx.needs_input_grad[4 + k]
            grads.append(torch.zeros_like(tb) if need else None)
        _lib.score_bwd(desc, h, r, t, gout.contiguous(), grads)
        return (None, None, None, None, *grads)


class RegFunction(torch.autograd.Function):
    """get_reg(h, r, t): lmbda * mean_b sum_rows g(x)  (pointwise.py:448-458,190-202,224-238)."""

    @staticmethod
    def forward(ctx, spec, reg_type, lmbda, h, r, t, *tables):
        _require_cuda(h, r, t, *tables)
        desc = spec.desc([tb.detach() for tb in tables])
        out = _lib.reg_fwd_bwd(desc, reg_type, lmbda, h.contiguous(), r.contiguous(), t.contiguous())
        ctx.spec, ctx.reg_type, ctx.lmbda = spec, reg_type, lmbda
        ctx.save_for_backward(h, r, t, *tables)
        return out.squeeze_(0)

    @staticmethod
    def backward(ctx, gout):
        h, r, t, *tables = ctx.saved_tensors
        desc = ctx.spec.desc([tb.detach() for tb in tables])
        grads = [torch.zeros_like(tb) for tb in tables]
        # d(reg)/d(table) scaled by the upstream scalar (read on the host: one tiny sync, as
        # loss.item() already is in the reference loop, trainer.py:300)
        _lib.reg_fwd_bwd(desc, ctx.reg_type, ctx.lmbda, h, r, t, grad_scale=float(gout), grad_tables=grads)
        return (None, None, None, None, None, None, *grads)


class HingeFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, neg, margin):
        _require_cuda(pos, neg)
        loss, gp, gn = _lib.loss_pairwise_hinge(pos.contiguous(), neg.contiguous(), float(margin))
        ctx.save_for_backward(gp, gn)
        return loss.squeeze_(0)   # in place: a VIEW returned from forward() may not be modified by the caller's `loss += reg` (trainer.py:155)

    @staticmethod
    def backward(ctx, g):
        gp, gn = ctx.saved_tensors
        return gp * g, gn * g, None


class LogisticFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, preds, target):
        _require_cuda(preds, target)
        loss, gpreds = _lib.loss_pointwise_logistic(preds.contiguous(), target.contiguous().float())
        ctx.save_for_backward(gpreds)
        return loss.squeeze_(0)   # in place: a VIEW returned from forward() may not be modified by the caller's `loss += reg` (trainer.py:155)

    @staticmethod
    def backward(ctx, g):
        (gpreds,) = ctx.saved_tensors
        return gpreds * g, None


class SelfAdvFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, neg, neg_rate, alpha):
        _require_cuda(pos, neg)
        loss, gp, gn = _lib.loss_selfadv(pos.contiguous(), neg.contiguous(), int(neg_rate), float(alpha))
        ctx.save_for_backward(gp, gn)
        return loss.squeeze_(0)   # in place: a VIEW returned from forward() may not be modified by the caller's `loss += reg` (trainer.py:155)

    @staticmethod
    def backward(ctx, g):
        gp, gn = ctx.saved_tensors
        return gp * g, gn * g, None, None


class ProjTailFunction(torch.autograd.Function):
    """preds [B,N] = sigmoid(x . E^T + b): the last layer of the projection models
    (projection.py:100-102).  Backward: kge_proj_tail_bwd (three tiled GEMM launches fused with
    the sigmoid derivative) — dense gradients for x, the entity table and the bias row."""

    @staticmethod
    def forward(ctx, x, ent, bias):
        _require_cuda(x, ent)
        x, ent_c = x.contiguous(), ent.contiguous()
        bias_c = bias.contiguous() if bias is not None else None
        preds = _lib.proj_tail_fwd(x.detach(), ent_c.detach(), bias_c.detach() if bias_c is not None else None)
        ctx.has_bias = bias is not None
        ctx.bias_shape = tuple(bias.shape) if bias is not None else None
        ctx.save_for_backward(x, ent_c, preds)
        return preds

    @staticmethod
    def backward(ctx, gpreds):
        x, ent, preds = ctx.saved_tensors
        gx = torch.zeros_like(x) if ctx.needs_input_grad[0] else None
        ge = torch.zeros_like(ent) if ctx.needs_input_grad[1] else None
        gb = torch.zeros(ent.shape[0], dtype=torch.float32, device=x.device) \
            if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        _lib.proj_tail_bwd(gpreds.contiguous(), preds, x.detach(), ent.detach(), gx, ge, gb)
        return gx, ge, (gb.reshape(ctx.bias_shape) if gb is not None else None)


class MultiClassBceFunction(torch.autograd.Function):
    """One direction of Criterion.multi_class_bce (criterion.py:41-50): value and d loss/d preds
    in one kernel (kge_proj_bce)."""

    @staticmethod
    def forward(ctx, preds, labels, label_scale, label_shift):
        _require_cuda(preds, labels)
        loss, g = _lib.proj_bce(preds.contiguous(), labels.contiguous().float(), float(label_scale),
                                float(label_shift), 1.0, want_grad=True)
        ctx.save_for_backward(g)
        return loss.squeeze_(0)   # in place: a VIEW returned from forward() may not be modified by the caller's `loss += reg` (trainer.py:155)

    @staticmethod
    def backward(ctx, gout):
        (g,) = ctx.saved_tensors
        return g * gout, None, None, None
