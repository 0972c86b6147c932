"""CPU tests (-m "not gpu"): the ProjE_pointwise oracle (tests/oracle_proje/kge_oracle_proje.c) against the golden
vectors the reference itself produced (tests/golden/make_golden_proje.py)."""
import numpy as np
import pytest

import oracle
import proje_util as pu


# (case, fp64): the fp64 path does not saturate where fp32 does (sigmoid rounds to 1 in fp32 only), so on the
# heavy case only the fp32 restatement follows the reference
STEP_CASES = [(n, False) for n in pu.CASES] + [(n, True) for n in pu.CASES if n != "proje_heavy"]


def _step(g, fp64):
    tabs = pu.tables(pu.state(g))
    loss, grads = pu.oracle_step(tabs, g["h"], g["r"], g["t"], g["lab_tail"], g["lab_head"],
                                 pu.noise_or_none(g, "tail"), pu.noise_or_none(g, "head"), fp64=fp64)
    reg = pu.oracle_reg(tabs, float(g["lmbda"]), grads)
    return loss, reg, grads


@pytest.mark.parametrize("name", pu.CASES)
def test_trunk_matches_reference(name):
    """f1 / f2: the only gap to the reference's x is tanh_canon against ATen's tanh"""
    g = pu.load(name)
    tabs = pu.tables(pu.state(g))
    for d, (tag, e) in enumerate((("tail", g["h"]), ("head", g["t"]))):
        assert np.abs(pu.oracle_trunk(tabs, e, g["r"], d) - g["x_" + tag]).max() <= 1e-6


@pytest.mark.parametrize("name,fp64", STEP_CASES)
def test_loss_and_regulariser_match_reference(name, fp64):
    g = pu.load(name)
    loss, reg, _ = _step(g, fp64)
    want_loss = float(g["loss_tail"]) + float(g["loss_head"])
    assert abs(loss - want_loss) <= 1e-5 * abs(want_loss)
    assert abs(reg - float(g["reg"])) <= 1e-5 * abs(float(g["reg"]))


@pytest.mark.parametrize("name,fp64", STEP_CASES)
def test_gradients_match_reference_autograd(name, fp64):
    """all eight gradients (step + get_reg), the bound the HypER training test uses: 5e-4 of the largest + 1e-7"""
    g = pu.load(name)
    _, _, grads = _step(g, fp64)
    for key, got, want in zip(pu.KEYS, grads, pu.golden_grads(g)):
        assert np.abs(got - want).max() <= 5e-4 * np.abs(want).max() + 1e-7, key


def test_heavy_case_exercises_both_clamps_and_ties():
    """the saturated case: sigmoid rounds to 1 (1 - s clamps to 1e-10) and falls below 1e-10 on labelled entries,
    and several entities tie at sigmoid = 1 for a query"""
    g = pu.load("proje_heavy")
    tabs = pu.tables(pu.state(g))
    _, _, logit, gg = pu.oracle_step(tabs, g["h"], g["r"], g["t"], g["lab_tail"], g["lab_head"], per_entry=True)
    lab = np.stack([g["lab_tail"], g["lab_head"]])
    s = 1.0 / (1.0 + np.exp(-logit[lab != 0].astype(np.float64)))
    assert (s < 1e-10).any() and (np.float32(s) == 1.0).any()
    assert (gg[lab != 0] == 0).any() and (gg[lab != 0] != 0).any()
    p = oracle.proj_tail_fwd(g["x_tail"], tabs[0], None)
    assert ((p == 1.0).sum(axis=1) > 1).any()


@pytest.mark.parametrize("name", pu.CASES)
def test_ranks_match_reference_evaluator(name):
    """count formulation over the oracle trunk == predict_*_rank + MetricCalculator, exactly"""
    g = pu.load(name)
    tabs = pu.tables(pu.state(g))
    Q = g["ranks"].shape[0]
    h, r, t = g["h"][:Q], g["r"][:Q], g["t"][:Q]
    c = np.zeros((Q, 4), dtype=np.int32)
    oracle.proj_rank(pu.oracle_trunk(tabs, h, r, 0), tabs[0], None, t, (g["filt_t_ptr"], g["filt_t_idx"]), 0, c)
    oracle.proj_rank(pu.oracle_trunk(tabs, t, r, 1), tabs[0], None, h, (g["filt_h_ptr"], g["filt_h_idx"]), 1, c)
    assert np.array_equal(c, g["ranks"])
