"""Helpers shared by the AcrE tests: the golden cases of tests/golden/make_golden_acre.py (stored under
golden/acre/), the reference state_dict as numpy (the int8 + scale weights expanded), the mirror built from it,
seeded reference-shaped states, and the CPU oracle of the inference trunk (tests/oracle_acre/kge_oracle_acre.c,
compiled here with gcc on first use)."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ACRE_DIR = os.path.join(HERE, "golden", "acre")
CASES = ["acre_serial_c4", "acre_parallel_c3"]
# (way, in_channels, atrous, acre_bias) at the FB15k-237 shape: hyperparams/AcrE.yaml's serial way, the CLI
# defaults (parallel, 9 channels), and the largest gate GEMM with distinct rates and no conv bias
FB237_CONFIGS = [("serial", 32, (1, 2, 2), True), ("parallel", 9, (1, 2, 2), True),
                 ("parallel", 32, (1, 3, 5), False)]
_ORACLE_SRC = os.path.join(HERE, "oracle_acre", "kge_oracle_acre.c")
_ORACLE_SO = os.path.join(HERE, "oracle_acre", "_build", "libkge_oracle_acre.so")
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


FIELDS = ("ent", "rel", "bn0_weight", "bn0_bias", "bn0_mean", "bn0_var", "conv1_weight", "conv1_bias",
          "conv2_weight", "conv2_bias", "conv3_weight", "conv3_bias", "W_gate_e_weight", "W_gate_e_bias",
          "bn1_weight", "bn1_bias", "bn1_mean", "bn1_var", "fc_weight", "fc_bias",
          "bn2_weight", "bn2_bias", "bn2_mean", "bn2_var")
KEYS = {"ent": "ent_embeddings.weight", "rel": "rel_embeddings.weight", "fc_weight": "fc.weight",
        "fc_bias": "fc.bias", "W_gate_e_weight": "W_gate_e.weight", "W_gate_e_bias": "W_gate_e.bias"}
for _l in ("conv1", "conv2", "conv3"):
    KEYS.update({_l + "_weight": _l + ".weight", _l + "_bias": _l + ".bias"})
for _bn in ("bn0", "bn1", "bn2"):
    KEYS.update({_bn + "_weight": _bn + ".weight", _bn + "_bias": _bn + ".bias",
                 _bn + "_mean": _bn + ".running_mean", _bn + "_var": _bn + ".running_var"})


class KgeAcre(ctypes.Structure):
    """kge_acre_t (include/kge_b200.h), as the oracle source declares it"""
    _fields_ = [("in_channels", ctypes.c_int32), ("way", ctypes.c_int32), ("first_atrous", ctypes.c_int32),
                ("second_atrous", ctypes.c_int32), ("third_atrous", ctypes.c_int32), ("hidden_size", ctypes.c_int32),
                ("num_rel", ctypes.c_int64),
                ("bn0_eps", ctypes.c_float), ("bn1_eps", ctypes.c_float), ("bn2_eps", ctypes.c_float)] + \
        [(n, ctypes.c_void_p) for n in FIELDS]


def config(state):
    """(way 0/1, in_channels, (atrous x3)) of a state: the states here carry it under "_config" """
    c = [int(v) for v in state["_config"]]
    return c[0], c[1], tuple(c[2:5])


def acre_struct(state, eps=1e-5):
    """-> (KgeAcre over host arrays, the arrays it points into: keep them alive while it is used)"""
    keep = {f: np.ascontiguousarray(state[k], dtype=np.float32) for f, k in KEYS.items() if k in state}
    way, C, atrous = config(state)
    p = KgeAcre()
    p.way, p.in_channels, p.hidden_size = way, C, keep["ent"].shape[1]
    p.first_atrous, p.second_atrous, p.third_atrous = atrous
    p.num_rel = keep["rel"].shape[0]
    p.bn0_eps = p.bn1_eps = p.bn2_eps = eps
    for f, a in keep.items():
        setattr(p, f, a.ctypes.data)
    return p, keep


def oracle_trunk_fwd(state, e, r, eps=1e-5, intermediates=False):
    """the oracle's AcrE trunk.  state: dict state_dict-key -> numpy array plus "_config"; e, r: ids (the head
    direction passes (t, r)).  -> x [Q, 200], or (x, feat [Q, C*400], gate [Q*C, 1600] or None) with
    intermediates=True."""
    p, keep = acre_struct(state, eps)
    e, r = np.ascontiguousarray(e, dtype=np.int64), np.ascontiguousarray(r, dtype=np.int64)
    Q, C = e.shape[0], p.in_channels
    x = np.empty((Q, 200), dtype=np.float32)
    feat = np.empty((Q, C * 400), dtype=np.float32) if intermediates else None
    gate = np.empty((Q * C, 1600), dtype=np.float32) if intermediates and p.way == 1 else None
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
    rc = oracle_lib().kgeo_acre_trunk_fwd(ctypes.byref(p), ptr(e), ptr(r), ctypes.c_int64(Q), ptr(x), ptr(feat),
                                          ptr(gate))
    assert rc == 0
    return (x, feat, gate) if intermediates else x


def load(name):
    return dict(np.load(os.path.join(ACRE_DIR, name + ".npz"), allow_pickle=False))


def state(g):
    """state_dict (numpy, in the reference's key order) of the reference AcrE stored in a case, plus its
    "_config"; the int8 + scale weights expanded exactly"""
    st = {}
    for key in g["sd_keys"]:
        key = str(key)
        st[key] = (g["q_" + key].astype(np.float32) * g["qscale_" + key]) if ("q_" + key) in g else g["sd_" + key]
    st["_config"] = np.array([g["way"], g["C"], *g["atrous"]])
    return st


def kwargs(way, C, atrous, bias, N, R, dropout=0.0, hidden_size=200):
    return dict(tot_entity=int(N), tot_relation=int(R), hidden_size=int(hidden_size), input_dropout=dropout,
                hidden_dropout=dropout, feature_map_dropout=dropout, in_channels=int(C),
                way=("serial" if way in (0, "serial") else "parallel"), first_atrous=int(atrous[0]),
                second_atrous=int(atrous[1]), third_atrous=int(atrous[2]), acre_bias=bool(bias))


def case_kwargs(g):
    return kwargs(int(g["way"]), int(g["C"]), g["atrous"], bool(g["acre_bias"]), g["N"], g["R"])


def mirror_from_state(st, N, R, device="cuda", train=False, dropout=0.0):
    """the package's AcrE with the given parameters / BN buffers (strict load)"""
    import torch
    from pykg2vec_b200 import import_model
    way, C, atrous = config(st)
    m = import_model("acre")(**kwargs(way, C, atrous, "conv1.bias" in st, N, R, dropout))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items() if k != "_config"}, strict=True)
    return m.to(device).train(train)


def mirror(g, device="cuda", train=False):
    return mirror_from_state(state(g), g["N"], g["R"], device, train)


def random_state(N, R, cfg, seed):
    """a reference-shaped AcrE state_dict (reference key order) with xavier tables, default-scale layers and
    non-trivial BN buffers / bias, as numpy.  cfg = (way, in_channels, atrous, acre_bias); R relations (the
    rel table has 2R rows, as in the reference)"""
    way, C, atrous, bias = cfg
    par = way in (1, "parallel")
    rng = np.random.RandomState(seed)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    unif = lambda shape, fan_in: f32(rng.uniform(-1, 1, shape) / np.sqrt(fan_in))
    xav = lambda rows, cols: f32(rng.uniform(-1, 1, (rows, cols)) * np.sqrt(6.0 / (rows + cols)))
    st = {"bias": f32(rng.standard_normal(N) * 0.3),
          "ent_embeddings.weight": xav(N, 200), "rel_embeddings.weight": xav(2 * R, 200)}
    for bn, n in (("bn0", 1), ("bn1", C), ("bn2", 200)):
        st[bn + ".weight"] = f32(rng.uniform(0.6, 1.4, n))
        st[bn + ".bias"] = f32(rng.standard_normal(n) * 0.2)
        st[bn + ".running_mean"] = f32(rng.standard_normal(n) * 0.2)
        st[bn + ".running_var"] = f32(rng.uniform(0.5, 1.5, n))
        st[bn + ".num_batches_tracked"] = np.array(0, dtype=np.int64)
    st["fc.weight"] = unif((200, C * 400), C * 400)
    st["fc.bias"] = unif(200, C * 400)
    for i, l in enumerate(("conv1", "conv2", "conv3")):
        cin = 1 if (par or i == 0) else C
        st[l + ".weight"] = unif((C, cin, 3, 3), 9 * cin)
        if bias:
            st[l + ".bias"] = unif(C, 9 * cin)
    if par:
        st["W_gate_e.weight"] = unif((400, 1600), 1600)
        st["W_gate_e.bias"] = unif(400, 1600)
    st["_config"] = np.array([1 if par else 0, C, *atrous])
    return st
