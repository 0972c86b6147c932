"""pykg2vec_b200 — H100-native (sm_90a) scoring engine behind pykg2vec's model surface.

Package layout (only what the hot path needs):
  csrc/        CUDA kernels + the C-ABI (include/kge_b200.h)  -> _build/libkge_b200.so
  _lib.py      ctypes binding of the C-ABI
  functional.py, criterion.py, KGMeta.py, Domain.py, pairwise.py, pointwise.py, projection.py
               host-side mirror of pykg2vec.models.* / pykg2vec.utils.criterion
  evaluator.py mirror of pykg2vec.utils.evaluator (batched 1-vs-all rank kernel)
  trainer.py   mirror of the Trainer hot loop (train_step_* + fused sparse steps)
  sharding.py  multi-GPU partitioning of the 1-vs-all evaluation
"""

# name -> (module, class): the targets pykg2vec.common.Importer.modelMap would point at
# (pykg2vec/common.py:266-297); see INTEGRATION.md.
MODEL_MAP = {
    "transe": ("pykg2vec_b200.pairwise", "TransE"),
    "transh": ("pykg2vec_b200.pairwise", "TransH"),
    "transd": ("pykg2vec_b200.pairwise", "TransD"),
    "transm": ("pykg2vec_b200.pairwise", "TransM"),
    "transr": ("pykg2vec_b200.pairwise", "TransR"),
    "rotate": ("pykg2vec_b200.pairwise", "RotatE"),
    "rescal": ("pykg2vec_b200.pairwise", "Rescal"),
    "hole": ("pykg2vec_b200.pairwise", "HoLE"),
    "kg2e": ("pykg2vec_b200.pairwise", "KG2E"),
    "slm": ("pykg2vec_b200.pairwise", "SLM"),
    "ntn": ("pykg2vec_b200.pairwise", "NTN"),
    "sme": ("pykg2vec_b200.pairwise", "SME"),
    "sme_bl": ("pykg2vec_b200.pairwise", "SME_BL"),
    "distmult": ("pykg2vec_b200.pointwise", "DistMult"),
    "cp": ("pykg2vec_b200.pointwise", "CP"),
    "complex": ("pykg2vec_b200.pointwise", "Complex"),
    "complexn3": ("pykg2vec_b200.pointwise", "ComplexN3"),
    "analogy": ("pykg2vec_b200.pointwise", "ANALOGY"),
    "quate": ("pykg2vec_b200.pointwise", "QuatE"),
    "octonione": ("pykg2vec_b200.pointwise", "OctonionE"),
    "simple": ("pykg2vec_b200.pointwise", "SimplE"),
    "simple_ignr": ("pykg2vec_b200.pointwise", "SimplE_ignr"),
    "convkb": ("pykg2vec_b200.pointwise", "ConvKB"),
    "conve": ("pykg2vec_b200.projection", "ConvE"),
    "tucker": ("pykg2vec_b200.projection", "TuckER"),
    "hyper": ("pykg2vec_b200.projection", "HypER"),
    "interacte": ("pykg2vec_b200.projection", "InteractE"),
    "acre": ("pykg2vec_b200.projection", "AcrE"),
    "proje_pointwise": ("pykg2vec_b200.projection", "ProjE_pointwise"),
}


def import_model(name):
    """Importer.import_model_config analogue (pykg2vec/common.py:300-325): returns the class."""
    import importlib
    try:
        mod, cls = MODEL_MAP[name.lower()]
    except KeyError:
        raise ValueError("%s model has not been implemented. please select from: %s"
                         % (name, ' '.join(sorted(MODEL_MAP))))
    return getattr(importlib.import_module(mod), cls)
