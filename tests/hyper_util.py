"""Helpers shared by the HypER tests: the golden cases of tests/golden/make_golden_hyper.py (stored under
golden/hyper/), the reference state_dict as numpy / torch, the mirror built from it, and the CPU oracle of
the inference trunk (tests/oracle_hyper/kge_oracle_hyper.c, compiled here with gcc on first use)."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
HYPER_DIR = os.path.join(HERE, "golden", "hyper")
CASES = ["hyper_d36", "hyper_d48"]
_ORACLE_SRC = os.path.join(HERE, "oracle_hyper", "kge_oracle_hyper.c")
_ORACLE_SO = os.path.join(HERE, "oracle_hyper", "_build", "libkge_oracle_hyper.so")
_oracle = None


def oracle_lib():
    """gcc -O2 -ffp-contract=off (no FMA contraction: fmaf() is explicit) + OpenMP, the flags of oracle/"""
    global _oracle
    if _oracle is None:
        if not os.path.exists(_ORACLE_SO) or os.path.getmtime(_ORACLE_SO) < os.path.getmtime(_ORACLE_SRC):
            os.makedirs(os.path.dirname(_ORACLE_SO), exist_ok=True)
            subprocess.run(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                            "-fopenmp", "-mfma", "-o", _ORACLE_SO + ".tmp", _ORACLE_SRC, "-lm"], check=True)
            os.replace(_ORACLE_SO + ".tmp", _ORACLE_SO)
        _oracle = ctypes.CDLL(_ORACLE_SO)
    return _oracle


HYPER_KEYS = {"ent": "ent_embeddings.weight", "rel": "rel_embeddings.weight", "fc1_weight": "fc1.weight",
              "fc1_bias": "fc1.bias", "fc_weight": "fc.weight", "fc_bias": "fc.bias"}
for _bn in ("bn0", "bn1", "bn2"):
    HYPER_KEYS.update({_bn + "_weight": _bn + ".weight", _bn + "_bias": _bn + ".bias",
                       _bn + "_mean": _bn + ".running_mean", _bn + "_var": _bn + ".running_var"})


class KgeHyper(ctypes.Structure):
    """kge_hyper_t (include/kge_b200.h), as the oracle source declares it"""
    _fields_ = [("ent_hidden_size", ctypes.c_int32), ("rel_hidden_size", ctypes.c_int32), ("num_rel", ctypes.c_int64),
                ("bn0_eps", ctypes.c_float), ("bn1_eps", ctypes.c_float), ("bn2_eps", ctypes.c_float)] + \
               [(n, ctypes.c_void_p) for n in ("ent", "rel", "bn0_weight", "bn0_bias", "bn0_mean", "bn0_var",
                                               "fc1_weight", "fc1_bias", "bn1_weight", "bn1_bias", "bn1_mean",
                                               "bn1_var", "fc_weight", "fc_bias", "bn2_weight", "bn2_bias",
                                               "bn2_mean", "bn2_var")]


def hyper_struct(state, eps=1e-5):
    """-> (KgeHyper over host arrays, the numpy arrays it points into: keep them alive while it is used)"""
    keep = {f: np.ascontiguousarray(state[k], dtype=np.float32) for f, k in HYPER_KEYS.items()}
    p = KgeHyper()
    p.ent_hidden_size, p.rel_hidden_size = keep["ent"].shape[1], keep["rel"].shape[1]
    p.num_rel = keep["rel"].shape[0]
    p.bn0_eps = p.bn1_eps = p.bn2_eps = eps
    for f, a in keep.items():
        setattr(p, f, a.ctypes.data)
    return p, keep


def oracle_trunk_fwd(state, e, r, eps=1e-5, intermediates=False):
    """the oracle's HypER trunk.  state: dict state_dict-key -> numpy array (the reference HypER's parameters and BN
    buffers); e, r: ids (the head direction passes (t, r): no reciprocal relations).  -> x [Q, de], or
    (x, filt [num_rel, 288], feat [Q, 32*(de-8)]) with intermediates=True."""
    p, keep = hyper_struct(state, eps)
    e, r = np.ascontiguousarray(e, dtype=np.int64), np.ascontiguousarray(r, dtype=np.int64)
    Q, de = e.shape[0], p.ent_hidden_size
    x = np.empty((Q, de), dtype=np.float32)
    filt = np.empty((p.num_rel, 288), dtype=np.float32) if intermediates else None
    feat = np.empty((Q, 32 * (de - 8)), dtype=np.float32) if intermediates else None
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
    rc = oracle_lib().kgeo_hyper_trunk_fwd(ctypes.byref(p), ptr(e), ptr(r), ctypes.c_int64(Q), ptr(x), ptr(filt),
                                           ptr(feat))
    assert rc == 0
    return (x, filt, feat) if intermediates else x


def load(name):
    return dict(np.load(os.path.join(HYPER_DIR, name + ".npz"), allow_pickle=False))


def state(g):
    """state_dict (numpy) of the reference HypER stored in a case"""
    return {k[3:]: g[k] for k in g if k.startswith("sd_") and not k.startswith("sd_after_")}


def kwargs(g, device="cuda"):
    return dict(tot_entity=int(g["N"]), tot_relation=int(g["R"]), ent_hidden_size=int(g["ent_hidden_size"]),
                rel_hidden_size=int(g["rel_hidden_size"]), input_dropout=0.0, hidden_dropout=0.0,
                feature_map_dropout=0.0, device=device)


def mirror(g, device="cuda", train=False):
    """the package's HypER with the reference's parameters and BN buffers (strict load)"""
    import torch
    from pykg2vec_b200 import import_model
    m = import_model("hyper")(**kwargs(g, device))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in state(g).items()}, strict=True)
    return m.to(device).train(train)


def random_state(N, R, de, dr, seed):
    """a reference-shaped HypER state_dict with xavier tables and non-trivial BN buffers / bias (numpy)"""
    rng = np.random.RandomState(seed)
    F = 32 * (de - 8)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    xav = lambda rows, cols: f32(rng.uniform(-1, 1, (rows, cols)) * np.sqrt(6.0 / (rows + cols)))
    st = {"b": f32(rng.standard_normal(N) * 0.3), "ent_embeddings.weight": xav(N, de),
          "rel_embeddings.weight": xav(R, dr),
          "fc.weight": f32(rng.uniform(-1, 1, (de, F)) / np.sqrt(F)), "fc.bias": f32(rng.uniform(-1, 1, de) / np.sqrt(F)),
          "fc1.weight": f32(rng.uniform(-1, 1, (288, dr)) / np.sqrt(dr)),
          "fc1.bias": f32(rng.uniform(-1, 1, 288) / np.sqrt(dr))}
    for bn, n in (("bn0", 1), ("bn1", 32), ("bn2", de)):
        st[bn + ".weight"] = f32(rng.uniform(0.6, 1.4, n))
        st[bn + ".bias"] = f32(rng.standard_normal(n) * 0.2)
        st[bn + ".running_mean"] = f32(rng.standard_normal(n) * 0.2)
        st[bn + ".running_var"] = f32(rng.uniform(0.5, 1.5, n))
        st[bn + ".num_batches_tracked"] = np.array(0, dtype=np.int64)
    return st
