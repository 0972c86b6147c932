"""Generator — device-side replacement of pykg2vec/data/generator.py (SURVEY.md §8f rank 1).

The reference feeds training from 1 feeder + `num_process_gen` sampler PROCESSES that build
negative batches with Python rejection loops (~1e4-1e5 triples/s/process) and ship them through
mp.Queues; at GPU scoring speed that pipeline is the bottleneck.  Here the training triples live
on the device, an epoch is a device permutation (raw_data_generator, generator.py:11-39), and
each batch's negatives are drawn by one kernel (kge_sample_negatives) against a device hash set
of the positives (process_function_pairwise / _pointwise, generator.py:42-158).

PROJECTION_BASED models (process_function_multiclass, generator.py:160-236) get their two dense
[batch, tot_entity] label matrices from one kernel per direction (kge_proj_labels) over device CSRs
of hr_t_train / tr_h_train: the reference assembles them per batch on the host with
torch.sparse(...).to_dense() and ships 2*B*N floats through the queue and over PCIe.  With neg_rate > 0
(ProjE_pointwise only) one device permutation per batch supplies the shared -1 negatives
(kge_proj_labels_negatives).

Same interface as the reference class: `Generator(model, config)`, `start_one_epoch(num_batch)`,
iteration yields the per-batch list (6 id arrays for pairwise, 4 for pointwise, [h, r, t, hr_t,
tr_h] for projection) — as DEVICE tensors, consumed by `Trainer.train_batch_device`.  `stop()` is
a no-op (no processes).
"""
import numpy as np
import torch

from . import _lib
from .KGMeta import TrainingStrategy


def relation_property(train, tot_relation):
    """KnowledgeGraph.read_relation_property (kgcontroller.py:466-492): per relation
    |distinct tails| / (|distinct heads| + |distinct tails|) over the training triples — the
    probability of corrupting the HEAD under Bernoulli sampling."""
    train = np.asarray(train)
    prob = np.zeros(tot_relation, dtype=np.float32)
    for r in range(tot_relation):
        sel = train[train[:, 1] == r]
        heads, tails = len(set(sel[:, 0].tolist())), len(set(sel[:, 2].tolist()))
        prob[r] = 0.0 if heads + tails == 0 else tails / (heads + tails)
    return prob


def _label_csr(known, first, rel, dev):
    """Device CSR of `known[(first, rel)]` over the distinct keys of the training triples, plus the
    CSR row of every training triple: (rows [n_train], ptr [K+1], idx [nnz]) int64 tensors."""
    keys, rows = {}, np.empty(len(first), dtype=np.int64)
    for i, key in enumerate(zip(first.tolist(), rel.tolist())):
        rows[i] = keys.setdefault(key, len(keys))
    ptr = np.zeros(len(keys) + 1, dtype=np.int64)
    chunks = []
    for key, row in keys.items():
        members = known[key]
        ptr[row + 1] = len(members)
        chunks.append(np.fromiter(members, dtype=np.int64, count=len(members)))
    np.cumsum(ptr, out=ptr)
    idx = np.concatenate(chunks) if chunks else np.zeros(0, dtype=np.int64)
    return tuple(torch.from_numpy(a).to(dev) for a in (rows, ptr, idx))


def negative_ids(num_ent, generator):
    """The shared negatives of one ProjE batch (process_function_multiclass with neg_rate > 0, generator.py:200-217):
    the first min(100, num_ent) ids of one random permutation of the entities, drawn on the generator's device.
    Every row of both directions gets -1 at these ids unless they are its positives."""
    return torch.randperm(int(num_ent), device=generator.device, generator=generator)[:min(100, int(num_ent))]


class Generator:
    def __init__(self, model, config, seed=0):
        self.model = model
        self.config = config
        self.training_strategy = model.training_strategy
        if self.training_strategy not in (TrainingStrategy.PAIRWISE_BASED, TrainingStrategy.POINTWISE_BASED,
                                          TrainingStrategy.PROJECTION_BASED):
            raise NotImplementedError("This strategy is not supported.")
        dev = torch.device(config.device)
        data = config.knowledge_graph.read_cache_data('triplets_train')
        arr = np.asarray([[t.h, t.r, t.t] for t in data], dtype=np.int64).reshape(-1, 3)
        self.train = torch.from_numpy(arr).to(dev)
        self._cols = [self.train[:, k].contiguous() for k in range(3)]
        self.slots = None
        self._negatives = False
        if self.training_strategy == TrainingStrategy.PROJECTION_BASED:
            if int(getattr(config, "neg_rate", 0)) > 0:
                if model.model_name.lower() != "proje_pointwise":
                    raise NotImplementedError("device label rows carry positives only (neg_rate must be 0, as in "
                                              "the ConvE / TuckER / InteractE / HypER / AcrE hyper-parameter files)")
                self._negatives = True   # ProjE: -1 labels at the batch's shared random negatives
            kgraph = config.knowledge_graph
            self._hr = _label_csr(kgraph.read_cache_data('hr_t_train'), arr[:, 0], arr[:, 1], dev)
            self._tr = _label_csr(kgraph.read_cache_data('tr_h_train'), arr[:, 2], arr[:, 1], dev)
        else:
            self.slots = _lib.tripleset_build(self._cols[0], self._cols[1], self._cols[2], config.tot_entity,
                                              config.tot_relation)
        self.head_prob = None
        if getattr(config, "sampling", "uniform") == "bern":
            self.head_prob = torch.from_numpy(relation_property(arr, config.tot_relation)).to(dev)
        self.seed = int(seed)
        self.step = 0
        self._perm = None
        self._remaining = 0
        self._batch_idx = 0
        self._gen = torch.Generator(device=dev)
        self._gen.manual_seed(self.seed)

    def __iter__(self):
        return self

    def start_one_epoch(self, num_batch):
        # one permutation per epoch, consumed in batch_size slices (generator.py:24,33-36)
        self._perm = torch.randperm(self.train.shape[0], device=self.train.device, generator=self._gen)
        self._remaining = int(num_batch)
        self._batch_idx = 0

    def __next__(self):
        if self._remaining <= 0:
            raise StopIteration
        B = self.config.batch_size
        sel = self._perm[self._batch_idx * B:(self._batch_idx + 1) * B]
        self._batch_idx += 1
        self._remaining -= 1
        ph, pr, pt = (c[sel] for c in self._cols)
        if self.training_strategy == TrainingStrategy.PROJECTION_BASED:
            n, N = int(sel.numel()), int(self.config.tot_entity)
            hr_t = _lib.proj_labels(self._hr[0][sel], self._hr[1], self._hr[2], n, N)
            tr_h = _lib.proj_labels(self._tr[0][sel], self._tr[1], self._tr[2], n, N)
            if self._negatives:
                neg = negative_ids(N, self._gen)
                _lib.proj_labels_negatives(hr_t, neg)
                _lib.proj_labels_negatives(tr_h, neg)
            self.step += 1
            return [ph, pr, pt, hr_t, tr_h]
        layout = 0 if self.training_strategy == TrainingStrategy.PAIRWISE_BASED else 1
        out = _lib.sample_negatives(self.slots, ph, pr, pt, int(self.config.neg_rate), self.head_prob,
                                    int(self.config.tot_entity), self.seed, self.step, layout=layout)
        self.step += 1
        if layout == 0:
            return [ph, pr, pt, out[0], out[1], out[2]]
        return list(out)

    def stop(self):
        return None
