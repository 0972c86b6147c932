"""Torch restatement of the reference's ATen op chains — TEST INFRASTRUCTURE ONLY.

Purpose (see oracle/__init__.py for the access rules):
  * fp64 autograd through these formulas is the GRADIENT oracle for the CUDA
    backward kernels (tests/);
  * fp32 on CPU with all host threads, it is the timed ``cpu_baseline`` /
    ``--impl reference`` arm of bench.py ("port": the real reference cannot travel
    to the GPU box).  It executes the same op sequence the reference does —
    gather, F.normalize, elementwise chain, reduction, full ``topk`` sort, D2H, and
    the per-triple Python rank walk — so its timing is representative of
    pykg2vec's own CPU path.

Every function cites the reference lines it follows (relative to /root/reference/).
It is pinned against the real reference by tests/test_oracle_golden.py.
"""
import math

import torch
import torch.nn.functional as F


def _norm_dist(h, r, t, l1):
    """pairwise.py:69-76 — normalise the three operands, then p-norm of h + r - t."""
    x = F.normalize(h, p=2, dim=-1) + F.normalize(r, p=2, dim=-1) - F.normalize(t, p=2, dim=-1)
    return torch.norm(x, p=1 if l1 else 2, dim=-1)


def score(name, tables, h, r, t, l1_flag=False, margin=0.0, embedding_range=None, rel_dim=None):
    """model.forward(h, r, t) for the in-scope models.  tables in C-ABI order
    (include/kge_b200.h, enum kge_model_id)."""
    name = name.lower()
    if name == "transe":  # pairwise.py:56-93
        ent, rel = tables
        return _norm_dist(ent[h], rel[r], ent[t], l1_flag)
    if name == "transm":  # pairwise.py:325-347
        ent, rel, theta = tables
        return theta[r] * _norm_dist(ent[h], rel[r], ent[t], l1_flag)
    if name == "transh":  # pairwise.py:143-182
        ent, rel, w = tables
        wn = F.normalize(w[r], p=2, dim=-1)
        eh, et = ent[h], ent[t]
        eh = eh - (eh * wn).sum(-1, keepdim=True) * wn
        et = et - (et * wn).sum(-1, keepdim=True) * wn
        return _norm_dist(eh, rel[r], et, l1_flag)
    if name == "transd":  # pairwise.py:229-278
        ent, rel, emap, rmap = tables
        eh, et, rm = ent[h], ent[t], rmap[r]
        eh = eh + (eh * emap[h]).sum(-1, keepdim=True) * rm
        et = et + (et * emap[t]).sum(-1, keepdim=True) * rm
        return _norm_dist(eh, rel[r], et, l1_flag)
    if name == "transr":  # pairwise.py:405-470
        ent, rel, mat = tables
        d = ent.shape[1]
        dr = rel.shape[1] if rel_dim is None else rel_dim
        eh = F.normalize(ent[h], p=2, dim=-1)
        er = F.normalize(rel[r], p=2, dim=-1)
        et = F.normalize(ent[t], p=2, dim=-1)
        m = mat[r].view(-1, d, dr)
        eh = torch.matmul(eh.unsqueeze(1), m).squeeze(1)
        et = torch.matmul(et.unsqueeze(1), m).squeeze(1)
        return _norm_dist(eh, er, et, l1_flag)
    if name == "rotate":  # pairwise.py:765-791
        ent_re, ent_im, rel = tables
        phase = rel[r] / (embedding_range / 3.14159265358979323846)
        re, im = torch.cos(phase), torch.sin(phase)
        hr, hi, tr, ti = ent_re[h], ent_im[h], ent_re[t], ent_im[t]
        sr = hr * re - hi * im - tr
        si = hr * im + hi * re - ti
        return -(margin - torch.sum(sr ** 2 + si ** 2, dim=-1))
    if name == "distmult":  # pointwise.py:444-446
        ent, rel = tables
        return -torch.sum(ent[h] * rel[r] * ent[t], -1)
    if name == "cp":  # pointwise.py:374-376
        sub, rel, obj = tables
        return -torch.sum(sub[h] * rel[r] * obj[t], -1)
    if name == "complex":  # pointwise.py:163-188
        ere, eim, rre, rim = tables
        hr, hi, tr, ti, rr, ri = ere[h], eim[h], ere[t], eim[t], rre[r], rim[r]
        return -torch.sum(hr * tr * rr + hi * ti * rr + hr * ti * ri - hi * tr * ri, -1)
    if name in ("slm", "ntn"):  # pairwise.py:525-541 / :919-960
        ent, rel, mr1, mr2 = tables[:4]
        nh, nr, nt = F.normalize(ent[h], p=2, dim=-1), F.normalize(rel[r], p=2, dim=-1), F.normalize(ent[t], p=2, dim=-1)
        pre = torch.matmul(nh, mr1) + torch.matmul(nt, mr2)
        if name == "ntn":
            br, mr = tables[4], tables[5]
            K, d = rel.shape[1], ent.shape[1]
            exp_h = nh.unsqueeze(0).repeat(K, 1, 1)
            temp = torch.matmul(exp_h, mr.view(K, d, d)).permute(1, 0, 2)
            htmrt = torch.squeeze(torch.matmul(temp, nt.unsqueeze(-1)), dim=-1)
            pre = htmrt + torch.matmul(nh, mr1) + torch.matmul(nt, mr2) + br
        return -torch.sum(nr * torch.tanh(pre), -1)
    if name in ("sme", "sme_bl"):  # pairwise.py:617-661 / :680-724
        ent, rel, mu1, mu2, bu, mv1, mv2, bv = tables
        nh, nr, nt = F.normalize(ent[h], p=2, dim=-1), F.normalize(rel[r], p=2, dim=-1), F.normalize(ent[t], p=2, dim=-1)
        u1, u2 = torch.matmul(mu1, nh.T), torch.matmul(mu2, nr.T)
        v1, v2 = torch.matmul(mv1, nt.T), torch.matmul(mv2, nr.T)
        if name == "sme":
            return -torch.sum((u1 + u2 + bu).T * (v1 + v2 + bv).T, 1)
        return torch.sum((u1 * u2 + bu).T * (v1 * v2 + bv).T, -1)
    if name == "kg2e":  # pairwise.py:1021-1084
        emu, esig, rmu, rsig = tables
        nrm = lambda x: x / torch.norm(x, 2, 1).view(-1, 1)
        hm, hs, rm, rs_, tm, ts = nrm(emu[h]), nrm(esig[h]), nrm(rmu[r]), nrm(rsig[r]), nrm(emu[t]), nrm(esig[t])
        cs, cm = hs + rs_, hm + rm
        return (cs / ts).sum(-1) + ((tm - cm) ** 2 / ts).sum(-1) + (torch.log(ts) - torch.log(cs)).sum(-1) - emu.shape[1]
    if name in ("quate", "octonione"):  # pointwise.py:678-694 / :886-899 (+ _qmult/_qstar/_omult/_onorm)
        C = 4 if name == "quate" else 8
        hc, tc = [tb[h] for tb in tables[:C]], [tb[t] for tb in tables[:C]]
        rc = [tb[r] for tb in tables[C:2 * C]]
        den = torch.sqrt(sum(x ** 2 for x in rc))
        rc = [x / den for x in rc]

        def qmult(a, b):
            return (a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                    a[0] * b[1] + b[0] * a[1] + a[2] * b[3] - b[2] * a[3],
                    a[0] * b[2] + b[0] * a[2] + a[3] * b[1] - b[3] * a[1],
                    a[0] * b[3] + b[0] * a[3] + a[1] * b[2] - b[1] * a[2])

        def star(a):
            return (a[0], -a[1], -a[2], -a[3])
        if C == 4:
            o = qmult(hc, rc)
        else:
            a, b, c, d_ = hc[:4], hc[4:], rc[:4], rc[4:]
            p1, p2 = qmult(a, c), qmult(star(d_), b)
            p3, p4 = qmult(d_, a), qmult(b, star(c))
            o = tuple(x - y for x, y in zip(p1, p2)) + tuple(x + y for x, y in zip(p3, p4))
        return -torch.sum(sum(x * y for x, y in zip(o, tc)), -1)
    if name == "analogy":  # pointwise.py:97-104
        ent, rel, ere, eim, rre, rim = tables
        hr, hi, tr, ti, rr, ri = ere[h], eim[h], ere[t], eim[t], rre[r], rim[r]
        cplx = -(hr * tr * rr + hi * ti * rr + hr * ti * ri - hi * tr * ri).sum(-1)
        dm = -(ent[h] * rel[r] * ent[t]).sum(-1)
        return cplx + dm
    if name == "rescal":  # pairwise.py:829-865, on tables already row-normalised by embed()
        ent, mat = tables
        d = ent.shape[1]
        m = mat[r].view(-1, d, d)
        return -torch.sum(ent[h].unsqueeze(2) * torch.matmul(m, ent[t].unsqueeze(2)), [1, 2])
    if name == "convkb_raw":
        # pointwise.py:302-318 as written.  tables = [ent, rel, conv_w0, conv_b0, conv_w1, conv_b1, ...,
        # fc_w, fc_b]: Conv2d(1->F,(3,w)) over the stacked [h;r;t] for every filter size, concat along
        # the width, flatten, Linear -> 1.
        ent, rel = tables[0], tables[1]
        fc_w, fc_b = tables[-2], tables[-1]
        x = torch.stack([ent[h], rel[r], ent[t]], dim=1).unsqueeze(1)          # [b,1,3,k]
        outs = [F.conv2d(x, tables[i], tables[i + 1]) for i in range(2, len(tables) - 2, 2)]
        flat = torch.cat(outs, dim=3).view(x.shape[0], -1)
        return torch.squeeze(F.linear(flat, fc_w, fc_b), dim=-1)
    if name == "convkb":
        # the same map in the collapsed affine form of the C-ABI (include/kge_b200.h KGE_CONVKB):
        # tables = [ent, rel, A(3 x k), c0(1)] from convkb_collapse() below
        ent, rel, A, c0 = tables
        return (ent[h] * A[0]).sum(-1) + (rel[r] * A[1]).sum(-1) + (ent[t] * A[2]).sum(-1) + c0[0]
    if name in ("simple", "simple_ignr"):  # pointwise.py:514-526, 573-581
        eh, et, rel, rinv = tables
        first = torch.sum(eh[h] * rel[r] * et[t], 1)
        second = torch.sum(eh[t] * rinv[r] * et[h], 1)
        init = first + second / 2.0 if name == "simple" else first + second
        return -torch.clamp(init, -20, 20)
    if name == "hole":
        # pairwise.py:1119-1125 as evaluated by torch<1.7 (legacy fft on [b,d,2] views, conj a no-op on
        # real tensors, elementwise product of the (re, im) pairs) -- see tests/golden/make_golden.py
        ent, rel = tables
        rn = F.normalize(rel[r], p=2, dim=-1)
        cdt = torch.complex128 if ent.dtype == torch.float64 else torch.complex64
        fh = torch.fft.fft(ent[h].to(cdt), dim=1)
        ft = torch.fft.fft(ent[t].to(cdt), dim=1)
        e = torch.fft.ifft(torch.complex(fh.real * ft.real, fh.imag * ft.imag), dim=1).real
        return -torch.sigmoid(torch.sum(rn * e, 1))
    raise NotImplementedError(name)


def convkb_collapse(conv_ws, conv_bs, fc_w, fc_b, k):
    """ConvKB has no nonlinearity between its convolutions and its Linear layer
    (pointwise.py:311-316), so score = <a_h,h> + <a_r,r> + <a_t,t> + c0 with
      A[row, j] = sum_w sum_f sum_q K_w[f,0,row,q] * W[f, off_w + j - q]   (0 <= j-q <= k-w)
      c0        = fc_b + sum_w sum_f b_w[f] * sum_p W[f, off_w + p]
    where W = fc_w.view(F, sum_w(k-w+1)) (concat along the width, then flatten: index f*sumP+off+p).
    Returns (A [3,k], c0 [1]) in the dtype of fc_w; differentiable w.r.t. every argument."""
    nf = conv_ws[0].shape[0]
    W = fc_w.reshape(nf, -1)
    A = torch.zeros((3, k), dtype=fc_w.dtype, device=fc_w.device)
    c0 = fc_b.reshape(1).clone()
    off = 0
    for kw_, kb_ in zip(conv_ws, conv_bs):
        w = kw_.shape[-1]
        P = k - w + 1
        Wf = W[:, off:off + P]                                   # [F, P]
        # out[row, j] = sum_f sum_q Wf[f, j-q] * K[f, row, q]
        A = A + F.conv_transpose1d(Wf.unsqueeze(0), kw_[:, 0]).squeeze(0)
        c0 = c0 + (kb_ * Wf.sum(1)).sum().reshape(1)
        off += P
    return A, c0


def gathered_rows(name, tables, h, r, t):
    """The rows get_reg() re-gathers (pointwise.py:448-458, 190-202, 377-388)."""
    name = name.lower()
    if name == "distmult":
        ent, rel = tables
        return [ent[h], rel[r], ent[t]]
    if name == "cp":
        sub, rel, obj = tables
        return [sub[h], rel[r], obj[t]]
    if name == "complex":
        ere, eim, rre, rim = tables
        return [ere[h], eim[h], rre[r], rim[r], ere[t], eim[t]]
    if name == "analogy":  # two groups with different widths (pointwise.py:106-119)
        ent, rel, ere, eim, rre, rim = tables
        return [ere[h], eim[h], rre[r], rim[r], ere[t], eim[t], ent[h], rel[r], ent[t]]
    raise NotImplementedError(name)


def reg(name, tables, h, r, t, lmbda, reg_type):
    """reg_type 0: F2 (x**2); 1: signed N3 (x**3, Complex/DistMult 'n3');
    2: |x|**3 (ComplexN3.get_reg, pointwise.py:224-238)."""
    if name.lower() in ("quate", "octonione"):  # pointwise.py:696-727 / :901-960: mean over [b, d] per table
        C = 4 if name.lower() == "quate" else 8
        rows = [tb[h] for tb in tables[:C]] + [tb[t] for tb in tables[:C]] + [tb[r] for tb in tables[C:2 * C]]
        p = 2 if reg_type == 0 else 3
        return lmbda * sum(torch.mean(torch.abs(x) ** p) for x in rows)
    rows = gathered_rows(name, tables, h, r, t)
    if reg_type == 0:
        per = sum(torch.sum(x ** 2, -1) for x in rows)
    elif reg_type == 1:
        per = sum(torch.sum(x ** 3, -1) for x in rows)
    else:
        per = sum(torch.sum(x.abs() ** 3, -1) for x in rows)
    return lmbda * torch.mean(per)


# ---- losses (pykg2vec/utils/criterion.py) -------------------------------------
def pairwise_hinge(pos, neg, margin):  # criterion.py:26-29
    v = pos + margin - neg
    return torch.max(v, torch.zeros_like(v)).sum()


def pointwise_logistic(preds, target):  # criterion.py:32-34
    return F.softplus(target * preds).mean()


def selfadv(pos, neg, neg_rate, alpha):  # criterion.py:14-23
    p = F.logsigmoid(-pos)
    n = (-neg).view(-1, neg_rate)
    w = torch.softmax(n * alpha, dim=1).detach()
    n = torch.sum(w * F.logsigmoid(-n), dim=-1)
    return -n.mean() - p.mean()


# ---- optimizer steps (torch.optim single-tensor update order, trainer.py:112-126) ----
# fp64 restatements of one dense step of the optimizers the trainer builds, with torch's defaults for every
# argument the trainer does not pass.  Arrays are float64 (numpy or torch); the hyperparameters are the float32
# values the kernels receive (kge_optim_apply_dense / kge_optim_apply_rows), widened exactly, so the only
# difference to the kernels is the rounding of each operation.  Each returns new arrays; the inputs are not changed.
def _f64(x):
    return x.double() if torch.is_tensor(x) else torch.from_numpy(x).double()


def sgd_step(w, g, lr):
    """torch.optim.SGD(lr): param.add_(grad, alpha=-lr).  Returns w'."""
    return _f64(w) - float(lr) * _f64(g)


def adagrad_step(w, g, state_sum, lr, eps=1e-10):
    """torch.optim.Adagrad(lr) (lr_decay 0, initial_accumulator_value 0): state_sum.addcmul_(grad, grad);
    std = state_sum.sqrt().add_(eps); param.addcdiv_(grad, std, value=-lr).  Returns (w', state_sum')."""
    g = _f64(g)
    s = _f64(state_sum) + g * g
    return _f64(w) - float(lr) * (g / (torch.sqrt(s) + float(eps))), s


def adam_step(w, g, exp_avg, exp_avg_sq, step, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    """torch.optim.Adam(lr) (no weight decay, no amsgrad) at step `step` >= 1:
    exp_avg.lerp_(grad, 1 - beta1); exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2);
    step_size = lr / (1 - beta1**step); denom = exp_avg_sq.sqrt() / sqrt(1 - beta2**step) + eps;
    param.addcdiv_(exp_avg, denom, value=-step_size).  Returns (w', exp_avg', exp_avg_sq')."""
    b1, b2 = float(beta1), float(beta2)
    g = _f64(g)
    m = _f64(exp_avg)
    m = m + (g - m) * (1.0 - b1)
    v = _f64(exp_avg_sq) * b2 + (1.0 - b2) * g * g
    step_size = float(lr) / (1.0 - b1 ** step)
    denom = torch.sqrt(v) / math.sqrt(1.0 - b2 ** step) + float(eps)
    return _f64(w) - step_size * (m / denom), m, v


# ---- evaluation (pykg2vec/utils/evaluator.py) ---------------------------------
def _walk(order, target, known):
    """MetricCalculator.get_tail_rank / get_head_rank, evaluator.py:70-123:
    read the descending-sorted id list from its END (best first) until the target."""
    rank = frank = 0
    for j in range(len(order)):
        e = order[-j - 1]
        if e == target:
            break
        rank += 1
        frank += 1
        if e in known:
            frank -= 1
    return rank, frank


def evaluate(score_fn, num_ent, triples, hr_t, tr_h, python_walk=True):
    """Evaluator.test, evaluator.py:309-334: per test triple two 1-vs-all forwards,
    a full topk(k=N) sort each, transfer to numpy, then the Python walk.
    score_fn(h, r, t) -> [b] scores for LongTensors.  Returns list of
    (trank, ftrank, hrank, fhrank) 0-based."""
    out = []
    ents = torch.arange(num_ent, dtype=torch.long)
    for (h, r, t) in triples:
        hb = torch.full((num_ent,), h, dtype=torch.long)
        rb = torch.full((num_ent,), r, dtype=torch.long)
        tb = torch.full((num_ent,), t, dtype=torch.long)
        _, head_order = torch.topk(score_fn(ents, rb, tb), k=num_ent)  # evaluator.py:262-273
        _, tail_order = torch.topk(score_fn(hb, rb, ents), k=num_ent)  # evaluator.py:249-260
        head_order = head_order.detach().cpu().numpy()
        tail_order = tail_order.detach().cpu().numpy()
        if python_walk:
            tr, ftr = _walk(tail_order, t, hr_t.get((h, r), ()))
            hrk, fhr = _walk(head_order, h, tr_h.get((t, r), ()))
            out.append((tr, ftr, hrk, fhr))
        else:
            out.append((int(tail_order[-1]), 0, int(head_order[-1]), 0))
    return out


def settle(ranks0, hits=(1, 3, 5, 10)):
    """MetricCalculator.settle, evaluator.py:125-141.  ranks0: [Q,4] 0-based
    (trank, ftrank, hrank, fhrank)."""
    import numpy as np
    a = np.asarray(ranks0)
    head = a[:, 2].astype(np.float32) + 1
    tail = a[:, 0].astype(np.float32) + 1
    fhead = a[:, 3].astype(np.float32) + 1
    ftail = a[:, 1].astype(np.float32) + 1
    ranks = np.concatenate((head, tail))
    franks = np.concatenate((fhead, ftail))
    res = {"mr": np.mean(ranks), "mrr": np.mean(np.reciprocal(ranks)),
           "fmr": np.mean(franks), "fmrr": np.mean(np.reciprocal(franks))}
    for k in hits:
        res["hit%d" % k] = np.mean(ranks <= k, dtype=np.float32)
        res["fhit%d" % k] = np.mean(franks <= k, dtype=np.float32)
    return res


def embedding_range(margin, dim):
    """RotatE.__init__, pairwise.py:748."""
    return (margin + 2.0) / dim


def xavier_uniform(rows, cols, gen):
    """nn.init.xavier_uniform_ on a [rows, cols] table (pairwise.py:46-47)."""
    a = math.sqrt(6.0 / (rows + cols))
    return (torch.rand(rows, cols, generator=gen, dtype=torch.float32) * 2 - 1) * a
