"""CPU tests (-m "not gpu") of the ProjE_pointwise mirror's host surface: constructor, state_dict layout,
parameter_list, seeded initialisation against the reference class, and the Generator's negative-id draw."""
import numpy as np
import pytest
import torch

import dropin_util as du
import proje_util as pu

KW = dict(tot_entity=40, tot_relation=6, hidden_size=12, lmbda=1e-5, hidden_dropout=0.5)


def test_constructor_surface_and_state_dict_layout():
    from pykg2vec_b200 import import_model
    P = import_model("ProjE_pointwise")
    with pytest.raises(Exception, match="hyperparameter hidden_dropout not found!"):
        P(**{k: v for k, v in KW.items() if k != "hidden_dropout"}, device="cpu")
    with pytest.raises(KeyError):       # the reference reads kwargs["device"] too
        P(**KW)
    m = P(**KW, device="cpu")
    assert m.model_name == "proje_pointwise" and m.training_strategy.name == "PROJECTION_BASED"
    assert m.device == "cpu" and m.loss.__name__ == "multi_class"
    assert list(m.state_dict()) == [k + ".weight" for k in pu.KEYS]
    assert [p.name for p in m.parameter_list] == ["ent_embedding", "rel_embedding", "bc1", "De1", "Dr1", "bc2", "De2",
                                                 "Dr2"]
    assert m.ent_embeddings.weight.shape == (40, 12) and m.rel_embeddings.weight.shape == (6, 12)
    assert all(getattr(m, k).weight.shape == (1, 12) for k in pu.KEYS[2:])
    assert m.proj_tail_tables()[1] is None
    with pytest.raises(AssertionError, match="Unknown forward direction"):
        m(torch.tensor([1]), torch.tensor([0]), torch.zeros(1, 40), direction="sideways")


@pytest.mark.parametrize("name", pu.CASES)
def test_golden_state_dict_loads_strictly(name):
    from pykg2vec_b200 import import_model
    g = pu.load(name)
    m = import_model("proje_pointwise")(**pu.kwargs(g, device="cpu"))
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in pu.state(g).items()}, strict=True)


@pytest.mark.skipif(not du.reference_available(), reason="oracle/_ref not installed (no reference checkout at build())")
def test_seeded_construction_draws_the_reference_weights():
    du.load_reference()
    from pykg2vec.models.projection import ProjE_pointwise as Ref
    from pykg2vec_b200 import import_model
    torch.manual_seed(11)
    ref = Ref(**KW, device="cpu")
    torch.manual_seed(11)
    own = import_model("proje_pointwise")(**KW, device="cpu")
    a, b = ref.state_dict(), own.state_dict()
    assert list(a) == list(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert [p.name for p in ref.parameter_list] == [p.name for p in own.parameter_list]


@pytest.mark.parametrize("N", [37, 100, 14541])
def test_negative_ids_are_min_100_distinct_entities(N):
    from pykg2vec_b200.generator import negative_ids
    gen = torch.Generator()
    gen.manual_seed(3)
    a = negative_ids(N, gen).numpy()
    assert len(a) == min(100, N) and len(set(a.tolist())) == len(a) and a.min() >= 0 and a.max() < N
    b = negative_ids(N, gen).numpy()      # a fresh permutation per batch
    assert N <= 1 or not np.array_equal(a, b)
