"""Helpers shared by the ConvE training-trunk tests: the golden cases of tests/golden/make_golden_conve_train.py (stored
under golden/conve_train/), the reference state as numpy, the CPU oracle (tests/oracle_conve_train/
kge_oracle_conve_train.c, compiled here with gcc on first use) and the reference's tail + loss in numpy fp64, which
turns the trunk's output into d loss / d x for the backward."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_DIR = os.path.join(HERE, "golden", "conve_train")
CASES = ["conve_train_k200_drop", "conve_train_12x6"]
PARAMS = ["ent_embeddings.weight", "rel_embeddings.weight", "bn0.weight", "bn0.bias", "conv2d_1.weight",
          "conv2d_1.bias", "bn1.weight", "bn1.bias", "fc.weight", "fc.bias", "bn2.weight", "bn2.bias"]
RUNNING = ["bn0.running_mean", "bn0.running_var", "bn1.running_mean", "bn1.running_var", "bn2.running_mean",
           "bn2.running_var"]
_ORACLE_SRC = os.path.join(HERE, "oracle_conve_train", "kge_oracle_conve_train.c")
_ORACLE_SO = os.path.join(HERE, "oracle_conve_train", "_build", "libkge_oracle_conve_train.so")
_oracle = None


def oracle_lib():
    """gcc -O2 -ffp-contract=off (no FMA contraction: fmaf() is explicit), the flags of oracle/"""
    global _oracle
    if _oracle is None:
        if not os.path.exists(_ORACLE_SO) or os.path.getmtime(_ORACLE_SO) < os.path.getmtime(_ORACLE_SRC):
            os.makedirs(os.path.dirname(_ORACLE_SO), exist_ok=True)
            subprocess.run(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                            "-mfma", "-o", _ORACLE_SO + ".tmp", _ORACLE_SRC, "-lm"], check=True)
            os.replace(_ORACLE_SO + ".tmp", _ORACLE_SO)
        _oracle = ctypes.CDLL(_ORACLE_SO)
    return _oracle


class KgeConveTrain(ctypes.Structure):
    """kge_conve_train_t (include/kge_b200.h), as the oracle and the emulation read it"""
    _fields_ = [("hidden_size", ctypes.c_int32), ("hidden_size_1", ctypes.c_int32)] + \
               [(n, ctypes.c_float) for n in ("bn0_eps", "bn1_eps", "bn2_eps", "bn0_momentum", "bn1_momentum",
                                              "bn2_momentum")] + \
               [(n, ctypes.c_void_p) for n in ("ent", "rel", "bn0_weight", "bn0_bias", "conv_weight", "conv_bias",
                                               "bn1_weight", "bn1_bias", "fc_weight", "fc_bias", "bn2_weight",
                                               "bn2_bias", "bn0_mean", "bn0_var", "bn1_mean", "bn1_var", "bn2_mean",
                                               "bn2_var")]


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def load(name):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False))
    k, h1 = int(g["hidden_size"]), int(g["hidden_size_1"])
    if "fc_seed" in g:   # the k = 200 case stores fc.weight as a numpy stream (make_golden_conve_train.py)
        F = 32 * (2 * (k // h1) - 2) * (h1 - 2)
        w = np.random.RandomState(int(g["fc_seed"])).standard_normal((k, F)) * g["fc_scale"]
        g["sd_fc.weight"] = w.astype(np.float32)
    return g


def state(g):
    """the reference's state_dict before the step, {key: numpy}"""
    return {k[3:]: np.asarray(v) for k, v in g.items() if k.startswith("sd_") and not k.startswith("sd_after_")}


def noises(g, tag):
    """(noise0 [b, 2k], noise1 [b, 32], noise2 [b, k]) the reference drew in the `tag` forward, or Nones"""
    if "noise0_" + tag not in g:
        return None, None, None
    return tuple(_f32(g["noise%d_%s" % (i, tag)]) for i in range(3))


def model_struct(sd, k, h1, running=True, eps=1e-5, momentum=0.1):
    """-> (KgeConveTrain over host copies of the state, {key: array} it points into: keep it alive while used).
    With running=True the struct's running statistics are COPIES that the forward updates in place."""
    keep = {key: np.array(sd[key], dtype=np.float32, copy=True) for key in PARAMS + RUNNING}
    p = KgeConveTrain()
    p.hidden_size, p.hidden_size_1 = k, h1
    p.bn0_eps = p.bn1_eps = p.bn2_eps = eps
    p.bn0_momentum = p.bn1_momentum = p.bn2_momentum = momentum
    names = ("ent", "rel", "bn0_weight", "bn0_bias", "conv_weight", "conv_bias", "bn1_weight", "bn1_bias",
             "fc_weight", "fc_bias", "bn2_weight", "bn2_bias")
    for n, key in zip(names, PARAMS):
        setattr(p, n, keep[key].ctypes.data)
    if running:
        for n, key in zip(("bn0_mean", "bn0_var", "bn1_mean", "bn1_var", "bn2_mean", "bn2_var"), RUNNING):
            setattr(p, n, keep[key].ctypes.data)
    return p, keep


def oracle_fwd(sd, k, h1, e, r, B, n0=None, n1=None, n2=None, running=None):
    """kgeo_conve_train_fwd -> x [Q, k]; `running` (a dict) receives the updated running statistics"""
    p, keep = model_struct(sd, k, h1)
    e, r, n0, n1, n2 = _i64(e), _i64(r), _f32(n0), _f32(n1), _f32(n2)
    x = np.full((len(e), k), np.nan, dtype=np.float32)
    oracle_lib().kgeo_conve_train_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B),
                                      _p(n0), _p(n1), _p(n2), _p(x))
    if running is not None:
        running.update({key: keep[key] for key in RUNNING})
    return x


def oracle_bwd64(sd, k, h1, e, r, B, gx, n0=None, n1=None, n2=None):
    """kgeo_conve_train_bwd64 -> ([12 fp64 gradients in PARAMS order], x64 [Q, k])"""
    p, keep = model_struct(sd, k, h1, running=False)
    e, r, n0, n1, n2 = _i64(e), _i64(r), _f32(n0), _f32(n1), _f32(n2)
    gx = np.ascontiguousarray(gx, dtype=np.float64)
    grads = [np.zeros(np.shape(sd[key]), dtype=np.float64) for key in PARAMS]
    arr = (ctypes.c_void_p * 12)(*[g.ctypes.data for g in grads])
    x64 = np.zeros((len(e), k), dtype=np.float64)
    oracle_lib().kgeo_conve_train_bwd64(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B),
                                        _p(n0), _p(n1), _p(n2), _p(gx), arr, _p(x64))
    return grads, x64


def tail_loss_and_grads(x, ent, bias, labels, smoothing, N):
    """one direction of the reference's tail + Criterion.multi_class_bce in fp64: (loss, d loss / d x, d ent, d b).
    The reference hands the predictions pr = sigmoid(x . E^T + b) to BCEWithLogitsLoss, which applies a second sigmoid
    (criterion.py:41-50, projection.py:100-102)."""
    x, ent, bias = np.asarray(x, np.float64), np.asarray(ent, np.float64), np.asarray(bias, np.float64).reshape(-1)
    pr = 1.0 / (1.0 + np.exp(-(x @ ent.T + bias)))
    y = (1.0 - smoothing) * np.asarray(labels, np.float64) + 1.0 / N
    loss = np.mean(np.maximum(pr, 0) - pr * y + np.log1p(np.exp(-np.abs(pr))))
    dz = (1.0 / (1.0 + np.exp(-pr)) - y) / pr.size * pr * (1.0 - pr)
    return loss, dz @ ent, dz.T @ x, dz.sum(0)


def golden_step(g, bwd=oracle_bwd64, fwd=oracle_fwd):
    """the reference's training step recomputed with the trunk of `fwd` / `bwd`: (loss, {param: gradient},
    {running key: value after both forwards}, x_tail, x_head)"""
    sd = state(g)
    k, h1, N, R = int(g["hidden_size"]), int(g["hidden_size_1"]), int(g["N"]), int(g["R"])
    B = len(g["h"])
    sm = float(g["label_smoothing"])
    run = {}
    loss, grads, xs = 0.0, {key: np.zeros(np.shape(v), np.float64) for key, v in sd.items()}, []
    for tag, e, r, lab in (("tail", g["h"], g["r"], g["lab_tail"]), ("head", g["t"], g["r"] + R, g["lab_head"])):
        nz = noises(g, tag)
        x = fwd(sd, k, h1, e, r, B, *nz, running=run)
        sd.update(run)   # the head forward starts from the running statistics the tail forward left
        xs.append(x)
        part, gx, gent, gb = tail_loss_and_grads(x, sd["ent_embeddings.weight"], sd["b.weight"], lab, sm, N)
        loss += part
        grads["ent_embeddings.weight"] += gent
        grads["b.weight"] += gb.reshape(grads["b.weight"].shape)
        trunk, _ = bwd(sd, k, h1, e, r, B, gx, *nz)
        for key, gr in zip(PARAMS, trunk):
            grads[key] += gr
    return loss, grads, run, xs[0], xs[1]


def golden_grad_check(g, grads, rel=5e-4, floor=1e-7):
    """every parameter's gradient against the reference's: the existing ConvE bound rel * max|want| + floor"""
    for key in [k[5:] for k in g if k.startswith("grad_")] + [k[11:] for k in g if k.startswith("gradsample_")]:
        got = np.asarray(grads[key])
        if "gradsample_" + key in g:
            got, want = got.reshape(-1)[::37], g["gradsample_" + key]
        else:
            want = g["grad_" + key]
        assert np.abs(got - want).max() <= rel * np.abs(want).max() + floor, key
