"""CPU tests (-m "not gpu"): the oracle's AcrE trunk restatement against the golden vectors the reference itself
produced (tests/golden/make_golden_acre.py), and the host surface of the AcrE mirror."""
import numpy as np
import pytest
import torch

import acre_util as au
import golden_util as gu
import oracle


@pytest.mark.parametrize("name", au.CASES)
def test_trunk_and_preds_match_reference(name):
    """trunk <= 1e-5 absolute, and trunk + tail within the 1e-4 relative bar on the predictions"""
    g = au.load(name)
    st = au.state(g)
    E, b = st["ent_embeddings.weight"], st["bias"]
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        x = au.oracle_trunk_fwd(st, e, g["r"])
        assert np.abs(x - g["x_" + tag]).max() <= 1e-5
        assert gu.rel_err(oracle.proj_tail_fwd(x, E, b), g["preds_" + tag]).max() <= 1e-4
        assert (x > 0).any() and (x == 0).any()


def _torch_trunk_fp64(st, e, r):
    """(gate input or None, features, x) of the reference's layers in torch CPU fp64 (conv2d with the rates)"""
    way, C, atrous = au.config(st)
    d = {k: torch.from_numpy(np.asarray(v)).double() for k, v in st.items() if v.dtype == np.float32}
    bn = lambda v, k, shape: ((v - d[k + ".running_mean"].view(shape)) / torch.sqrt(d[k + ".running_var"].view(shape) + 1e-5)
                              * d[k + ".weight"].view(shape) + d[k + ".bias"].view(shape))
    conv = lambda x, l, a: torch.nn.functional.conv2d(x, d[l + ".weight"], d.get(l + ".bias"), 1, a, a)
    img = torch.cat([d["ent_embeddings.weight"][torch.from_numpy(e)].view(-1, 1, 10, 20),
                     d["rel_embeddings.weight"][torch.from_numpy(r)].view(-1, 1, 10, 20)], 2)
    img = bn(img, "bn0", (1, 1, 1, 1))
    gate = None
    if way == 0:
        y = conv(conv(conv(img, "conv1", atrous[0]), "conv2", atrous[1]), "conv3", atrous[2]) + img
    else:
        parts = [img.expand(-1, C, 20, 20).reshape(-1, C, 400)] + \
            [conv(img, l, a).reshape(-1, C, 400) for l, a in zip(("conv1", "conv2", "conv3"), atrous)]
        gate = torch.cat(parts, 2)
        y = (gate @ d["W_gate_e.weight"].T + d["W_gate_e.bias"]).view(-1, C, 20, 20)
        gate = gate.reshape(-1, 1600)
    feat = torch.relu(bn(y, "bn1", (1, C, 1, 1))).reshape(len(e), -1)
    x = torch.relu(bn(feat @ d["fc.weight"].T + d["fc.bias"], "bn2", (1, -1)))
    return gate, feat, x


@pytest.mark.parametrize("name", au.CASES)
def test_each_stage_follows_the_reference_layers(name):
    """the gate input (parallel), the features relu(bn1(.)) and x each match the reference's layers in fp64"""
    g = au.load(name)
    st = au.state(g)
    x, feat, gate = au.oracle_trunk_fwd(st, g["h"], g["r"], intermediates=True)
    wgate, wfeat, wx = _torch_trunk_fp64(st, g["h"], g["r"])
    if gate is not None:
        assert np.abs(gate - wgate.numpy()).max() <= 1e-5
    assert np.abs(feat - wfeat.numpy()).max() <= 1e-5
    assert np.abs(x - wx.numpy()).max() <= 1e-5


@pytest.mark.parametrize("cfg", [("serial", 3, (20, 1, 37), False), ("parallel", 2, (25, 19, 1), True)])
def test_rates_at_and_beyond_the_image(cfg):
    """rates >= 20 leave only the centre tap inside the image; the oracle still follows the reference's layers"""
    st = au.random_state(30, 4, cfg, seed=9)
    e, r = np.array([0, 5, 29]), np.array([0, 7, 3])
    x, feat, gate = au.oracle_trunk_fwd(st, e, r, intermediates=True)
    _, wfeat, wx = _torch_trunk_fp64(st, e, r)
    assert np.abs(feat - wfeat.numpy()).max() <= 1e-5 and np.abs(x - wx.numpy()).max() <= 1e-5


@pytest.mark.parametrize("name", au.CASES)
@pytest.mark.parametrize("own_trunk", [False, True])
def test_ranks_match_reference_evaluator(name, own_trunk):
    """count formulation == the reference's predict_*_rank + MetricCalculator walk, exactly"""
    g = au.load(name)
    st = au.state(g)
    Q = g["ranks"].shape[0]
    h, r, t = g["h"][:Q], g["r"][:Q], g["t"][:Q]
    if own_trunk:
        xt, xh = au.oracle_trunk_fwd(st, h, r), au.oracle_trunk_fwd(st, t, r)
    else:
        xt, xh = g["x_tail"][:Q], g["x_head"][:Q]
    E, b = st["ent_embeddings.weight"], st["bias"]
    c = np.zeros((Q, 4), dtype=np.int32)
    oracle.proj_rank(xt, E, b, t, (g["filt_t_ptr"], g["filt_t_idx"]), 0, c)
    oracle.proj_rank(xh, E, b, h, (g["filt_h_ptr"], g["filt_h_idx"]), 1, c)
    assert np.array_equal(c, g["ranks"])


@pytest.mark.parametrize("name", au.CASES)
def test_training_loss_restated_from_stored_preds(name):
    """the stored train-mode loss is Criterion.multi_class_bce of the stored predictions (oracle BCE)"""
    g = au.load(name)
    N = int(g["N"])
    scale, shift = np.float32(1.0 - float(g["label_smoothing"])), np.float32(1.0 / N)
    total = sum(oracle.proj_bce(g["tr_preds_" + tag], g["tr_labels_" + tag], scale, shift, 1.0)[0]
                for tag in ("tail", "head"))
    assert abs(total - float(g["tr_loss"])) <= 2e-6 * abs(total)


# ---- host surface of the mirror (no GPU, no compute) ---------------------------------------------
@pytest.mark.parametrize("name", au.CASES)
def test_mirror_state_dict_is_the_reference_layout(name):
    from pykg2vec_b200 import import_model
    g = au.load(name)
    st = {k: v for k, v in au.state(g).items() if k != "_config"}
    m = import_model("acre")(**au.case_kwargs(g))
    own = m.state_dict()
    assert list(own) == list(st)          # same keys in the same order
    mods = [k.split(".")[0] for k in own]
    order = list(dict.fromkeys(mods))
    want = ["bias", "ent_embeddings", "rel_embeddings", "bn0", "bn1", "bn2", "fc", "conv1", "conv2", "conv3"]
    assert order == want + (["W_gate_e"] if int(g["way"]) == 1 else [])
    assert ("conv1.bias" in own) == bool(g["acre_bias"])
    for k, v in st.items():
        assert tuple(own[k].shape) == tuple(v.shape), k
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    assert [p.name for p in m.parameter_list] == ["ent_embedding", "rel_embedding"]
    assert m.model_name == "acre" and m.training_strategy.name == "PROJECTION_BASED"
    assert m.ent_embeddings.padding_idx is None and m.rel_embeddings.padding_idx is None
    assert m.rel_embeddings.weight.shape == (2 * int(g["R"]), 200)
    assert m.loss.__name__ == "multi_class_bce"
    assert m.get_reg(None, None, None) == 0.0
    for l, a in zip(("conv1", "conv2", "conv3"), g["atrous"]):
        conv = getattr(m, l)
        assert conv.dilation == (a, a) and conv.padding == (a, a) and conv.kernel_size == (3, 3)


@pytest.mark.parametrize("name", au.CASES)
def test_seeded_construction_equals_the_reference(name):
    """with the reference's torch seed the mirror draws the same initial weights (the fixture keeps ent / rel /
    conv* / small biases as constructed, and fc.weight / W_gate_e.weight as a sample of entries + row sums)"""
    from pykg2vec_b200 import import_model
    g = au.load(name)
    seed = int(g["seed"])
    np.random.seed(seed)
    torch.manual_seed(seed)
    m = import_model("acre")(**au.case_kwargs(g))
    own = {k: v.numpy() for k, v in m.state_dict().items()}
    for key in own:
        if key.startswith(("ent_", "rel_", "conv")) or key in ("fc.bias", "W_gate_e.bias"):
            assert np.array_equal(own[key], g["sd_" + key]), key
    for key in ("fc.weight", "W_gate_e.weight"):
        if "init_idx_" + key not in g:
            assert key not in own
            continue
        assert np.array_equal(own[key].reshape(-1)[g["init_idx_" + key]], g["init_sample_" + key]), key
        assert np.array_equal(own[key].astype(np.float64).sum(1), g["init_rowsum_" + key]), key
    assert not own["bias"].any()
    for bn in ("bn0", "bn1", "bn2"):
        assert (own[bn + ".weight"] == 1).all() and not own[bn + ".bias"].any()
        assert not own[bn + ".running_mean"].any() and (own[bn + ".running_var"] == 1).all()


def test_golden_fixtures_stay_small_and_exact():
    """each fixture is under 1 MB; the int8 weights times their power-of-two scale are exact fp32 values"""
    import os
    for name in au.CASES:
        assert os.path.getsize(os.path.join(au.ACRE_DIR, name + ".npz")) < (1 << 20)
        g = au.load(name)
        for key in ("fc.weight", "W_gate_e.weight"):
            if "q_" + key in g:
                assert g["q_" + key].dtype == np.int8 and np.abs(g["q_" + key]).max() <= 7
                assert float(g["qscale_" + key]) == 2.0 ** -8


def test_mirror_contract_errors():
    from pykg2vec_b200 import import_model, _lib
    A = import_model("AcrE")
    kw = au.kwargs("serial", 2, (1, 2, 2), True, 10, 3)
    for missing in ("in_channels", "way", "acre_bias", "third_atrous", "hidden_size"):
        with pytest.raises(Exception, match="hyperparameter %s not found!" % missing):
            A(**{k: v for k, v in kw.items() if k != missing})
    m = A(**dict(kw, hidden_size=100))          # constructs whatever the size, as upstream
    assert m.fc.weight.shape == (100, 800)
    m = A(**dict(kw, way="other"))              # the reference's test: anything but "serial" is parallel
    assert hasattr(m, "W_gate_e") and m.conv2.weight.shape == (2, 1, 3, 3)
    e, r = torch.tensor([1, 0]), torch.tensor([0, 2])
    with pytest.raises(AssertionError, match="Unknown forward direction"):
        m(e, r, direction="sideways")
    with pytest.raises(_lib.KgeError, match="no CPU"):      # no CPU fallback for the product path
        m(e, r, direction="tail")


@pytest.mark.parametrize("way", ["serial", "parallel"])
def test_training_layers_run_on_cpu_tensors(way):
    """the training trunk (the reference's layers) itself is device-agnostic: gradients reach every conv"""
    from pykg2vec_b200 import import_model
    torch.manual_seed(0)
    m = import_model("acre")(**au.kwargs(way, 3, (1, 3, 5), True, 20, 4)).train()
    x = m._trunk_layers(torch.tensor([1, 5, 0, 7]), torch.tensor([0, 3, 2, 7]))
    assert x.shape == (4, 200)
    x.sum().backward()
    for l in ("conv1", "conv2", "conv3"):
        assert getattr(m, l).weight.grad.abs().sum() > 0, l
