"""Drop-in proof (SURVEY.md §8b): the REFERENCE's own Importer -> Trainer.build_model / train_model -> Evaluator
-> infer_* flow (scripts/pykg2vec_train.py:11-23) runs unchanged with this package's classes patched into
Importer.modelMap, and a checkpoint written by the reference loads into them.

BASELINE.json configs[0] (`pykg2vec-train -mn TransE -ds umls`, CPU plumbing) is served by the UNMODIFIED
reference classes — the product has no CPU path by design (a CPU fallback would void every parity claim);
test_config1_cli_flow_reference_cpu runs exactly that flow here on the UMLS-shaped synthetic dataset, and
the -m gpu test runs the same flow through this package's classes with `-device cuda`.  Both need the
unmodified reference that build() installs under oracle/_ref/ (oracle/reference.py) and skip without it.

The checkpoint test needs nothing outside the repository: a slice of the reference's
examples/pretrained/TransE/model.vec.pt (FB15k, d=50, L1) and the reference's scores on it are stored in
golden/pretrained_transe_fb15k_slice.npz (golden/make_golden.py)."""
import numpy as np
import pytest
import torch

import dropin_util as du
import golden_util as gu

needs_ref = pytest.mark.skipif(not du.reference_available(), reason="oracle/_ref not installed (no reference checkout at build())")
CFG1 = ["-mn", "TransE", "-l", "2", "-ts", "1", "-tn", "50", "-npg", "1"]   # defaults otherwise: d=50, B=128, adam, L1, margin 0.8


def _flow(tmp_path, monkeypatch, extra, importer_cls=None):
    du.load_reference()
    ds = du.write_dataset(str(tmp_path / "data"))
    monkeypatch.chdir(tmp_path)   # the reference creates ../dataset relative to the CWD (datasets.py:84-86)
    return du.run_cli_flow(CFG1 + ["-ds", "syn", "-dsp", ds] + extra, importer_cls)


@needs_ref
def test_config1_cli_flow_reference_cpu(tmp_path, monkeypatch):
    """configs[0]: the reference CLI flow on CPU with its own classes (what `-device cpu` keeps using)."""
    tr = _flow(tmp_path, monkeypatch, ["-device", "cpu"])
    assert type(tr.model).__module__ == "pykg2vec.models.pairwise"
    assert len(tr.training_results) == 2 and np.isfinite(tr.training_results[-1][1])
    mc = tr.evaluator.metric_calculator
    assert len(mc.mr) >= 1 and all(np.isfinite(v) for v in mc.mr.values())


@needs_ref
@pytest.mark.gpu
@pytest.mark.parametrize("model,extra", [("TransE", []), ("DistMult", []), ("Complex", []),
                                         ("RotatE", ["-ngr", "4"]), ("TransH", []), ("Rescal", ["-k", "16"])])
def test_reference_trainer_drives_b200_classes(tmp_path, monkeypatch, model, extra):
    """the unmodified reference Trainer / Generator / Evaluator with this package's model classes, -device cuda"""
    B200Importer = du.b200_importer_class()
    du.load_reference()
    ds = du.write_dataset(str(tmp_path / "data"))
    monkeypatch.chdir(tmp_path)
    argv = ["-mn", model, "-l", "2", "-ts", "1", "-tn", "50", "-npg", "1", "-ds", "syn", "-dsp", ds, "-device", "cuda"] + extra
    tr = du.run_cli_flow(argv, B200Importer)
    assert type(tr.model).__module__.startswith("pykg2vec_b200.")
    assert next(tr.model.parameters()).is_cuda
    assert len(tr.training_results) == 2 and np.isfinite(tr.training_results[-1][1])
    # loss goes down on the training set between the two epochs (the kernels really train the tables)
    assert tr.training_results[1][1] < tr.training_results[0][1]
    mc = tr.evaluator.metric_calculator
    assert all(np.isfinite(v) for v in mc.mr.values())
    # Trainer.infer_* (trainer.py:330-386) through the reference's Evaluator.test_*_rank
    assert len(tr.infer_tails(1, 10, topk=5)) == 5
    assert len(tr.infer_heads(10, 20, topk=5)) == 5
    # the reference's ranks over this package's forward == the batched rank kernel on the same weights
    from pykg2vec_b200.evaluator import Evaluator as B200Evaluator
    ev = B200Evaluator(tr.model, tr.config)
    ev.full_test(epoch=0)
    ref_mc = tr.evaluator.metric_calculator
    tr.model.eval()
    with torch.no_grad():
        tr.evaluator.full_test(0)
    got = np.stack([ev.metric_calculator.rank_tail, ev.metric_calculator.rank_head], axis=1)
    want = np.stack([ref_mc.rank_tail, ref_mc.rank_head], axis=1)
    # identical except where torch.topk's order under exact ties decides (count them: must be rare)
    assert (got != want).mean() < 0.02, (got != want).mean()


@pytest.mark.gpu
def test_pretrained_checkpoint_loads_like_the_reference(tmp_path):
    """the checkpoint slice loads the way Trainer.load_model loads a checkpoint (`model.load_state_dict(
    torch.load(path))`, pykg2vec/utils/trainer.py:399-419) and scores like the reference's own TransE."""
    import pykg2vec_b200
    g = gu.load("pretrained_transe_fb15k_slice")
    n_ent, n_rel = g["table0"].shape[0], g["table1"].shape[0]
    path = tmp_path / "model.vec.pt"
    torch.save({"ent_embeddings.weight": torch.from_numpy(g["table0"]),
                "rel_embeddings.weight": torch.from_numpy(g["table1"])}, str(path))
    m = pykg2vec_b200.import_model("TransE")(tot_entity=n_ent, tot_relation=n_rel, hidden_size=int(g["kw_hidden_size"]),
                                             l1_flag=bool(g["kw_l1_flag"]))
    m.load_state_dict(torch.load(str(path), map_location="cpu"))
    assert type(m).__module__ == "pykg2vec_b200.pairwise" and m.ent_embeddings.weight.shape == (n_ent, 50)
    m = m.cuda()
    with torch.no_grad():
        got = m(*(torch.from_numpy(g[k]).cuda() for k in ("h", "r", "t"))).cpu().numpy()
    want = g["scores"]
    err = np.abs(got - want) / np.maximum(np.abs(want), 1e-2 * np.abs(want).max())
    assert err.max() < 1e-4, err.max()
