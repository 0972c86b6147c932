"""Helpers shared by the InteractE tests: the golden cases of tests/golden/make_golden_interacte.py (stored under
golden/interacte/), the reference state_dict as numpy, the mirror built from it (with the stored chequer
permutation), seeded reference-shaped states, and the CPU oracle of the inference trunk
(tests/oracle_interacte/kge_oracle_interacte.c, compiled here with gcc on first use)."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
INTERACTE_DIR = os.path.join(HERE, "golden", "interacte")
CASES = ["interacte_p2", "interacte_p3"]
# the three distinct FB15k-237-shaped configurations of hyperparams/InteractE.yaml: (P, F, ks, rh, rw)
YAML_CONFIGS = [(1, 96, 9, 20, 10), (2, 96, 11, 20, 10), (4, 64, 7, 20, 10)]
_ORACLE_SRC = os.path.join(HERE, "oracle_interacte", "kge_oracle_interacte.c")
_ORACLE_SO = os.path.join(HERE, "oracle_interacte", "_build", "libkge_oracle_interacte.so")
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


FIELDS = ("ent", "rel", "bn0_weight", "bn0_bias", "bn0_mean", "bn0_var", "conv_filt", "bn1_weight", "bn1_bias",
          "bn1_mean", "bn1_var", "fc_weight", "fc_bias", "bn2_weight", "bn2_bias", "bn2_mean", "bn2_var")
KEYS = {"ent": "ent_embeddings.weight", "rel": "rel_embeddings.weight", "conv_filt": "conv_filt",
        "fc_weight": "fc.weight", "fc_bias": "fc.bias"}
for _bn in ("bn0", "bn1", "bn2"):
    KEYS.update({_bn + "_weight": _bn + ".weight", _bn + "_bias": _bn + ".bias",
                 _bn + "_mean": _bn + ".running_mean", _bn + "_var": _bn + ".running_var"})


class KgeInteracte(ctypes.Structure):
    """kge_interacte_t (include/kge_b200.h), as the oracle source declares it"""
    _fields_ = [("feature_permutation", ctypes.c_int32), ("num_filters", ctypes.c_int32),
                ("kernel_size", ctypes.c_int32), ("reshape_height", ctypes.c_int32),
                ("reshape_width", ctypes.c_int32), ("num_rel", ctypes.c_int64),
                ("bn0_eps", ctypes.c_float), ("bn1_eps", ctypes.c_float), ("bn2_eps", ctypes.c_float),
                ("perm", ctypes.c_void_p)] + [(n, ctypes.c_void_p) for n in FIELDS]


def geometry(state):
    """(P, F, ks, reshape_height, reshape_width) of a state: the reshape is not recoverable from the tensor shapes,
    so the states here carry the geometry under "_geometry" """
    return tuple(int(v) for v in state["_geometry"])


def interacte_struct(state, perm, eps=1e-5):
    """-> (KgeInteracte over host arrays, the arrays it points into: keep them alive while it is used)"""
    keep = {f: np.ascontiguousarray(state[k], dtype=np.float32) for f, k in KEYS.items()}
    keep["perm"] = np.ascontiguousarray(perm, dtype=np.int64)
    P, F, ks, rh, rw = geometry(state)
    p = KgeInteracte()
    p.feature_permutation, p.num_filters, p.kernel_size, p.reshape_height, p.reshape_width = P, F, ks, rh, rw
    p.num_rel = keep["rel"].shape[0]
    p.bn0_eps = p.bn1_eps = p.bn2_eps = eps
    for f, a in keep.items():
        setattr(p, f, a.ctypes.data)
    return p, keep


def oracle_trunk_fwd(state, perm, e, r, eps=1e-5, intermediates=False):
    """the oracle's InteractE trunk.  state: dict state_dict-key -> numpy array plus "_geometry"; perm: the chequer
    permutation [P, 2k]; e, r: ids (the head direction passes (t, r): no reciprocal relations).  -> x [Q, k], or
    (x, feat [Q, P*F*H*W]) with intermediates=True."""
    p, keep = interacte_struct(state, perm, eps)
    e, r = np.ascontiguousarray(e, dtype=np.int64), np.ascontiguousarray(r, dtype=np.int64)
    Q, k = e.shape[0], p.reshape_height * p.reshape_width
    x = np.empty((Q, k), dtype=np.float32)
    Fw = p.feature_permutation * p.num_filters * 2 * k
    feat = np.empty((Q, Fw), dtype=np.float32) if intermediates else None
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
    rc = oracle_lib().kgeo_interacte_trunk_fwd(ctypes.byref(p), ptr(e), ptr(r), ctypes.c_int64(Q), ptr(x), ptr(feat))
    assert rc == 0
    return (x, feat) if intermediates else x


def load(name):
    return dict(np.load(os.path.join(INTERACTE_DIR, name + ".npz"), allow_pickle=False))


def state(g):
    """state_dict (numpy) of the reference InteractE stored in a case, plus its "_geometry" """
    st = {k[3:]: g[k] for k in g if k.startswith("sd_") and not k.startswith("sd_after_")}
    st["_geometry"] = np.array([g["P"], g["F"], g["ks"], g["reshape_height"], g["reshape_width"]])
    return st


def kwargs(geom, N, R, device="cuda", dropout=0.0):
    P, F, ks, rh, rw = geom
    return dict(tot_entity=int(N), tot_relation=int(R), hidden_size=int(rh * rw), input_dropout=dropout,
                hidden_dropout=dropout, feature_map_dropout=dropout, feature_permutation=int(P), num_filters=int(F),
                kernel_size=int(ks), reshape_height=int(rh), reshape_width=int(rw), device=device)


def case_kwargs(g, device="cuda"):
    return kwargs(geometry(state(g)), g["N"], g["R"], device)


def mirror_from_state(st, perm, N, R, device="cuda", train=False, dropout=0.0):
    """the package's InteractE with the given parameters / BN buffers (strict load) and chequer permutation"""
    import torch
    from pykg2vec_b200 import import_model
    m = import_model("interacte")(**kwargs(geometry(st), N, R, device, dropout))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items() if k != "_geometry"}, strict=True)
    m.chequer_perm = torch.from_numpy(np.asarray(perm, dtype=np.int64)).to(device)
    return m.to(device).train(train)


def mirror(g, device="cuda", train=False):
    return mirror_from_state(state(g), g["chequer_perm"], g["N"], g["R"], device, train)


def random_state(N, R, geom, seed):
    """(a reference-shaped InteractE state_dict with xavier tables and non-trivial BN buffers / bias, a random
    chequer-like permutation [P, 2k]) as numpy"""
    P, F, ks, rh, rw = geom
    k = rh * rw
    Fw = P * F * 2 * k
    rng = np.random.RandomState(seed)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    xav = lambda rows, cols: f32(rng.uniform(-1, 1, (rows, cols)) * np.sqrt(6.0 / (rows + cols)))
    st = {"bias": f32(rng.standard_normal(N) * 0.3),
          "conv_filt": f32(rng.uniform(-1, 1, (F, 1, ks, ks)) * np.sqrt(6.0 / (ks * ks * (1 + F)))),
          "ent_embeddings.weight": xav(N, k), "rel_embeddings.weight": xav(R, k)}
    for bn, n in (("bn0", P), ("bn1", P * F), ("bn2", k)):
        st[bn + ".weight"] = f32(rng.uniform(0.6, 1.4, n))
        st[bn + ".bias"] = f32(rng.standard_normal(n) * 0.2)
        st[bn + ".running_mean"] = f32(rng.standard_normal(n) * 0.2)
        st[bn + ".running_var"] = f32(rng.uniform(0.5, 1.5, n))
        st[bn + ".num_batches_tracked"] = np.array(0, dtype=np.int64)
    st["fc.weight"] = f32(rng.uniform(-1, 1, (k, Fw)) / np.sqrt(Fw))
    st["fc.bias"] = f32(rng.uniform(-1, 1, k) / np.sqrt(Fw))
    st["_geometry"] = np.array(geom)
    perm = np.stack([rng.permutation(2 * k) for _ in range(P)]).astype(np.int64)
    return st, perm
