"""Shared by the drop-in tests: the reference's own CLI flow (scripts/pykg2vec_train.py:11-23) on a
UMLS-shaped synthetic dataset, with or without this package's classes patched into Importer.  The reference is
the unmodified package build() installs under oracle/_ref/ (oracle/reference.py)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def reference_available():
    from baseline import ref_loader
    from oracle import reference
    return ref_loader.available(reference.REF_DIR)


def load_reference():
    from baseline import ref_loader
    from oracle import reference
    return ref_loader.load(reference.REF_DIR)


def write_dataset(dirpath, name="syn", n_ent=135, n_rel=46, n_train=5216, n_valid=652, n_test=661, seed=0):
    """<name>-train.txt / -valid.txt / -test.txt, tab separated (pykg2vec/data/datasets.py:374-431);
    UMLS statistics by default (BASELINE.json configs[0]; the real files cannot be downloaded offline)."""
    rng = np.random.RandomState(seed)
    os.makedirs(dirpath, exist_ok=True)
    ents = ["e%03d" % i for i in range(n_ent)]
    rels = ["r%02d" % i for i in range(n_rel)]
    first = True
    for split, n in (("train", n_train), ("valid", n_valid), ("test", n_test)):
        h, r, t = rng.randint(n_ent, size=n), rng.randint(n_rel, size=n), rng.randint(n_ent, size=n)
        if first:   # every entity / relation occurs in the training split
            h[:n_ent], t[:n_ent] = np.arange(n_ent), np.arange(n_ent)[::-1]
            r[:n_rel] = np.arange(n_rel)
            first = False
        with open(os.path.join(dirpath, "%s-%s.txt" % (name, split)), "w") as f:
            for a, b, c in zip(h, r, t):
                f.write("%s\t%s\t%s\n" % (ents[a], rels[b], ents[c]))
    return dirpath


def b200_importer_class():
    """The maintainer's patch of INTEGRATION.md §2 as a subclass: the in-scope names resolve under
    pykg2vec_b200 instead of pykg2vec.models (pykg2vec/common.py:266-325) — two attributes change."""
    load_reference()
    from pykg2vec.common import Importer
    import pykg2vec_b200

    class B200Importer(Importer):
        def __init__(self):
            super().__init__()
            self.model_path = "pykg2vec_b200"
            self.modelMap = {name: "%s.%s" % (mod.split(".")[-1], cls) for name, (mod, cls) in pykg2vec_b200.MODEL_MAP.items()}
    return B200Importer


def run_cli_flow(argv, importer_cls=None):
    """scripts/pykg2vec_train.py main(), verbatim, with the Importer class injectable.  Returns the trainer."""
    load_reference()
    from pykg2vec.common import Importer, KGEArgParser
    from pykg2vec.data.kgcontroller import KnowledgeGraph
    from pykg2vec.utils.trainer import Trainer
    args = KGEArgParser().get_args(argv)
    knowledge_graph = KnowledgeGraph(dataset=args.dataset_name, custom_dataset_path=args.dataset_path)
    knowledge_graph.prepare_data()
    config_def, model_def = (importer_cls or Importer)().import_model_config(args.model_name.lower())
    config = config_def(args)
    model = model_def(**config.__dict__)
    trainer = Trainer(model, config)
    trainer.build_model()
    trainer.train_model()
    return trainer
