"""CPU tests (-m "not gpu"): the oracle's HypER trunk restatement against the golden vectors the reference
itself produced (tests/golden/make_golden_hyper.py), and the host surface of the HypER mirror."""
import numpy as np
import pytest
import torch

import golden_util as gu
import hyper_util as hu
import oracle


@pytest.mark.parametrize("name", hu.CASES)
def test_trunk_and_preds_match_reference(name):
    """trunk <= 1e-5 absolute, and trunk + tail within the 1e-4 relative bar on the predictions"""
    g = hu.load(name)
    st = hu.state(g)
    E, b = st["ent_embeddings.weight"], st["b"]
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        x = hu.oracle_trunk_fwd(st, e, g["r"])
        assert np.abs(x - g["x_" + tag]).max() <= 1e-5
        assert gu.rel_err(oracle.proj_tail_fwd(x, E, b), g["preds_" + tag]).max() <= 1e-4
        # the reference's own x through the oracle tail: the tail alone is ~1e-7 away
        assert gu.rel_err(oracle.proj_tail_fwd(g["x_" + tag], E, b), g["preds_" + tag]).max() < 1e-6


@pytest.mark.parametrize("name", hu.CASES)
def test_intermediates_follow_the_reference_layers(name):
    """the filter table is fc1(rel) and the features are bn1(conv) of the reference's layers (torch CPU, fp64)"""
    g = hu.load(name)
    st = hu.state(g)
    x, filt, feat = hu.oracle_trunk_fwd(st, g["h"], g["r"], intermediates=True)
    d = {k: torch.from_numpy(np.asarray(v)).double() for k, v in st.items() if v.dtype == np.float32}
    want_filt = d["rel_embeddings.weight"] @ d["fc1.weight"].T + d["fc1.bias"]
    assert np.abs(filt - want_filt.numpy()).max() <= 1e-6
    bn = lambda v, k, shape: ((v - d[k + ".running_mean"].view(shape)) / torch.sqrt(d[k + ".running_var"].view(shape) + 1e-5)
                              * d[k + ".weight"].view(shape) + d[k + ".bias"].view(shape))
    v = bn(d["ent_embeddings.weight"][torch.from_numpy(g["h"])], "bn0", (1, 1))
    w = want_filt[torch.from_numpy(g["r"])].view(-1, 32, 9)
    de = v.shape[1]
    conv = torch.stack([sum(w[:, c, t, None] * v[:, t:t + de - 8] for t in range(9)) for c in range(32)], 1)
    want_feat = bn(conv, "bn1", (1, 32, 1)).reshape(len(g["h"]), -1)     # no ReLU, channel-major
    assert np.abs(feat - want_feat.numpy()).max() <= 1e-5
    want_x = torch.relu(bn(torch.from_numpy(feat).double() @ d["fc.weight"].T + d["fc.bias"], "bn2", (1, -1)))
    assert np.abs(x - want_x.numpy()).max() <= 1e-5


@pytest.mark.parametrize("name", hu.CASES)
@pytest.mark.parametrize("own_trunk", [False, True])
def test_ranks_match_reference_evaluator(name, own_trunk):
    """count formulation == the reference's predict_*_rank + MetricCalculator walk, exactly"""
    g = hu.load(name)
    st = hu.state(g)
    Q = g["ranks"].shape[0]
    h, r, t = g["h"][:Q], g["r"][:Q], g["t"][:Q]
    if own_trunk:
        xt, xh = hu.oracle_trunk_fwd(st, h, r), hu.oracle_trunk_fwd(st, t, r)
    else:
        xt, xh = g["x_tail"][:Q], g["x_head"][:Q]
    E, b = st["ent_embeddings.weight"], st["b"]
    c = np.zeros((Q, 4), dtype=np.int32)
    oracle.proj_rank(xt, E, b, t, (g["filt_t_ptr"], g["filt_t_idx"]), 0, c)
    oracle.proj_rank(xh, E, b, h, (g["filt_h_ptr"], g["filt_h_idx"]), 1, c)
    assert np.array_equal(c, g["ranks"])


@pytest.mark.parametrize("name", hu.CASES)
def test_training_loss_restated_from_stored_preds(name):
    """the stored train-mode loss is Criterion.multi_class_bce of the stored predictions (oracle BCE)"""
    g = hu.load(name)
    N = int(g["N"])
    scale, shift = np.float32(1.0 - float(g["label_smoothing"])), np.float32(1.0 / N)
    total = sum(oracle.proj_bce(g["tr_preds_" + tag], g["tr_labels_" + tag], scale, shift, 1.0)[0]
                for tag in ("tail", "head"))
    assert abs(total - float(g["tr_loss"])) <= 2e-6 * abs(total)


# ---- host surface of the mirror (no GPU, no compute) ---------------------------------------------
@pytest.mark.parametrize("name", hu.CASES)
def test_hyper_mirror_state_dict_is_the_reference_layout(name):
    from pykg2vec_b200 import import_model
    g = hu.load(name)
    st = hu.state(g)
    m = import_model("hyper")(**hu.kwargs(g, device="cpu"))
    own = m.state_dict()
    assert list(own) == list(st)          # same keys in the same order
    for k, v in st.items():
        assert tuple(own[k].shape) == tuple(v.shape), k
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    assert [p.name for p in m.parameter_list] == ["ent_embeddings", "rel_embeddings"]
    assert m.model_name == "hyper" and m.training_strategy.name == "PROJECTION_BASED"
    assert m.ent_embeddings.padding_idx == 0 and m.rel_embeddings.padding_idx == 0
    assert m.loss.__name__ == "multi_class_bce" and m.device == "cpu"
    assert m.get_reg(None, None, None) == 0.0


def test_hyper_mirror_contract_errors():
    from pykg2vec_b200 import import_model, _lib
    H = import_model("HypER")
    kw = dict(tot_entity=10, tot_relation=3, ent_hidden_size=12, rel_hidden_size=6, input_dropout=0.0,
              hidden_dropout=0.0, feature_map_dropout=0.0)
    with pytest.raises(Exception, match="hyperparameter rel_hidden_size not found!"):
        H(**{k: v for k, v in kw.items() if k != "rel_hidden_size"}, device="cpu")
    with pytest.raises(KeyError):       # the reference reads kwargs["device"] too
        H(**kw)
    m = H(**kw, device="cpu")
    e, r = torch.tensor([1, 0]), torch.tensor([0, 2])
    with pytest.raises(AssertionError, match="Unknown forward direction"):
        m(e, r, direction="sideways")
    with pytest.raises(_lib.KgeError, match="no CPU"):      # no CPU fallback for the product path
        m(e, r, direction="tail")


def test_padding_rows_get_no_lookup_gradient():
    """padding_idx=0: the lookup gradient of row 0 is zero (the reference's nn.Embedding semantics)"""
    from pykg2vec_b200 import import_model
    m = import_model("hyper")(tot_entity=10, tot_relation=3, ent_hidden_size=12, rel_hidden_size=6, input_dropout=0.0,
                              hidden_dropout=0.0, feature_map_dropout=0.0, device="cpu")
    e, r = torch.tensor([0, 3, 0]), torch.tensor([0, 2, 1])
    (m.ent_embeddings(e).sum() + m.rel_embeddings(r).sum()).backward()
    assert not m.ent_embeddings.weight.grad[0].any() and m.ent_embeddings.weight.grad[3].all()
    assert not m.rel_embeddings.weight.grad[0].any() and m.rel_embeddings.weight.grad[2].all()
