"""CPU tests (-m "not gpu"): the oracle's InteractE trunk restatement against the golden vectors the reference
itself produced (tests/golden/make_golden_interacte.py), and the host surface of the InteractE mirror."""
import numpy as np
import pytest
import torch

import golden_util as gu
import interacte_util as iu
import oracle


@pytest.mark.parametrize("name", iu.CASES)
def test_trunk_and_preds_match_reference(name):
    """trunk <= 1e-5 absolute, and trunk + tail within the 1e-4 relative bar on the predictions"""
    g = iu.load(name)
    st = iu.state(g)
    E, b = st["ent_embeddings.weight"], st["bias"]
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        x = iu.oracle_trunk_fwd(st, g["chequer_perm"], e, g["r"])
        assert np.abs(x - g["x_" + tag]).max() <= 1e-5
        assert gu.rel_err(oracle.proj_tail_fwd(x, E, b), g["preds_" + tag]).max() <= 1e-4
        assert (x > 0).any() and (x == 0).any()


@pytest.mark.parametrize("name", iu.CASES)
def test_features_follow_the_reference_layers(name):
    """the features are relu(bn1(circular conv)) of the reference's layers (torch CPU, fp64)"""
    g = iu.load(name)
    st = iu.state(g)
    P, F, ks, rh, rw = iu.geometry(st)
    H, W, pad = 2 * rw, rh, ks // 2
    x, feat = iu.oracle_trunk_fwd(st, g["chequer_perm"], g["h"], g["r"], intermediates=True)
    d = {k: torch.from_numpy(np.asarray(v)).double() for k, v in st.items() if v.dtype == np.float32}
    bn = lambda v, k, shape: ((v - d[k + ".running_mean"].view(shape)) / torch.sqrt(d[k + ".running_var"].view(shape) + 1e-5)
                              * d[k + ".weight"].view(shape) + d[k + ".bias"].view(shape))
    comb = torch.cat([d["ent_embeddings.weight"][torch.from_numpy(g["h"])],
                      d["rel_embeddings.weight"][torch.from_numpy(g["r"])]], 1)
    img = bn(comb[:, torch.from_numpy(g["chequer_perm"])].reshape(-1, P, H, W), "bn0", (1, P, 1, 1))
    img = torch.nn.functional.pad(img, (pad, pad, pad, pad), mode="circular")
    conv = torch.nn.functional.conv2d(img, d["conv_filt"].repeat(P, 1, 1, 1), groups=P)
    want_feat = torch.relu(bn(conv, "bn1", (1, P * F, 1, 1))).reshape(len(g["h"]), -1)
    assert np.abs(feat - want_feat.numpy()).max() <= 1e-5
    want_x = torch.relu(bn(torch.from_numpy(feat).double() @ d["fc.weight"].T + d["fc.bias"], "bn2", (1, -1)))
    assert np.abs(x - want_x.numpy()).max() <= 1e-5


@pytest.mark.parametrize("name", iu.CASES)
@pytest.mark.parametrize("own_trunk", [False, True])
def test_ranks_match_reference_evaluator(name, own_trunk):
    """count formulation == the reference's predict_*_rank + MetricCalculator walk, exactly"""
    g = iu.load(name)
    st = iu.state(g)
    Q = g["ranks"].shape[0]
    h, r, t = g["h"][:Q], g["r"][:Q], g["t"][:Q]
    if own_trunk:
        xt, xh = iu.oracle_trunk_fwd(st, g["chequer_perm"], h, r), iu.oracle_trunk_fwd(st, g["chequer_perm"], t, r)
    else:
        xt, xh = g["x_tail"][:Q], g["x_head"][:Q]
    E, b = st["ent_embeddings.weight"], st["bias"]
    c = np.zeros((Q, 4), dtype=np.int32)
    oracle.proj_rank(xt, E, b, t, (g["filt_t_ptr"], g["filt_t_idx"]), 0, c)
    oracle.proj_rank(xh, E, b, h, (g["filt_h_ptr"], g["filt_h_idx"]), 1, c)
    assert np.array_equal(c, g["ranks"])


@pytest.mark.parametrize("name", iu.CASES)
def test_training_loss_restated_from_stored_preds(name):
    """the stored train-mode loss is Criterion.multi_class_bce of the stored predictions (oracle BCE)"""
    g = iu.load(name)
    N = int(g["N"])
    scale, shift = np.float32(1.0 - float(g["label_smoothing"])), np.float32(1.0 / N)
    total = sum(oracle.proj_bce(g["tr_preds_" + tag], g["tr_labels_" + tag], scale, shift, 1.0)[0]
                for tag in ("tail", "head"))
    assert abs(total - float(g["tr_loss"])) <= 2e-6 * abs(total)


# ---- host surface of the mirror (no GPU, no compute) ---------------------------------------------
@pytest.mark.parametrize("name", iu.CASES)
def test_mirror_state_dict_is_the_reference_layout(name):
    from pykg2vec_b200 import import_model
    g = iu.load(name)
    st = {k: v for k, v in iu.state(g).items() if k != "_geometry"}
    m = import_model("interacte")(**iu.case_kwargs(g, device="cpu"))
    own = m.state_dict()
    assert list(own) == list(st)          # same keys in the same order
    assert list(own)[:4] == ["bias", "conv_filt", "ent_embeddings.weight", "rel_embeddings.weight"]
    for k, v in st.items():
        assert tuple(own[k].shape) == tuple(v.shape), k
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    assert [p.name for p in m.parameter_list] == ["ent_embeddings", "rel_embeddings"]
    assert m.model_name == "interacte" and m.training_strategy.name == "PROJECTION_BASED"
    assert m.ent_embeddings.padding_idx is None and m.rel_embeddings.padding_idx is None
    assert m.loss.__name__ == "multi_class_bce" and m.device == "cpu"
    assert isinstance(m.bceloss, torch.nn.BCELoss)
    assert m.hidden_size == int(g["reshape_height"]) * int(g["reshape_width"])
    assert "chequer_perm" not in own and not any(t is m.chequer_perm for t in m.buffers())
    assert m.get_reg(None, None, None) == 0.0


@pytest.mark.parametrize("name", iu.CASES)
def test_seeded_construction_equals_the_reference(name):
    """with the reference's numpy and torch seeds the mirror draws the same chequer permutation and the same
    initial ent / rel / conv_filt / fc (the fixture keeps those as constructed; BN and bias were set afterwards)"""
    from pykg2vec_b200 import import_model
    g = iu.load(name)
    seed = int(g["seed"])
    np.random.seed(seed)
    torch.manual_seed(seed)
    m = import_model("interacte")(**iu.case_kwargs(g, device="cpu"))
    assert m.chequer_perm.dtype == torch.int64 and tuple(m.chequer_perm.shape) == g["chequer_perm"].shape
    assert np.array_equal(m.chequer_perm.numpy(), g["chequer_perm"])
    own = m.state_dict()
    for key in ("ent_embeddings.weight", "rel_embeddings.weight", "conv_filt", "fc.weight", "fc.bias"):
        assert np.array_equal(own[key].numpy(), g["sd_" + key]), key
    assert not own["bias"].any()
    for bn in ("bn0", "bn1", "bn2"):
        assert (own[bn + ".weight"] == 1).all() and not own[bn + ".bias"].any()
        assert not own[bn + ".running_mean"].any() and (own[bn + ".running_var"] == 1).all()
    # every image holds each entity and each relation feature exactly once
    k = m.hidden_size
    for row in m.chequer_perm.numpy():
        assert np.array_equal(np.sort(row), np.arange(2 * k))


def test_mirror_contract_errors():
    from pykg2vec_b200 import import_model, _lib
    I = import_model("InteractE")
    kw = iu.kwargs((2, 4, 3, 4, 3), 10, 3, device="cpu")
    with pytest.raises(Exception, match="hyperparameter num_filters not found!"):
        I(**{k: v for k, v in kw.items() if k != "num_filters"})
    with pytest.raises(Exception, match="hyperparameter hidden_size not found!"):   # required, then overwritten
        I(**{k: v for k, v in kw.items() if k != "hidden_size"})
    with pytest.raises(KeyError):       # the reference reads kwargs["device"] too
        I(**{k: v for k, v in kw.items() if k != "device"})
    m = I(**dict(kw, hidden_size=999))
    assert m.hidden_size == 12 and m.ent_embeddings.weight.shape == (10, 12)
    e, r = torch.tensor([1, 0]), torch.tensor([0, 2])
    with pytest.raises(AssertionError, match="Unknown forward direction"):
        m(e, r, direction="sideways")
    with pytest.raises(_lib.KgeError, match="no CPU"):      # no CPU fallback for the product path
        m(e, r, direction="tail")


def test_training_layers_run_on_cpu_tensors():
    """the training trunk (the reference's layers) itself is device-agnostic: gradients reach conv_filt"""
    from pykg2vec_b200 import import_model
    torch.manual_seed(0)
    m = import_model("interacte")(**iu.kwargs((3, 4, 5, 6, 4), 20, 4, device="cpu")).train()
    x = m._trunk_layers(torch.tensor([1, 5, 0, 7]), torch.tensor([0, 3, 2, 1]))
    assert x.shape == (4, 24)
    x.sum().backward()
    assert m.conv_filt.grad is not None and m.conv_filt.grad.abs().sum() > 0
