"""Trainer hot loop — mirror of the per-batch part of pykg2vec/utils/trainer.py
(build_model optimizer selection :103-144, train_step_pairwise :147-157,
train_step_pointwise :176-180, and the batch body of train_model_epoch :269-300).

Two execution modes for the same step semantics:
  * autograd mode (any torch optimizer, e.g. adam): model(...) / model.loss(...) /
    loss.backward() / optimizer.step() exactly as the reference Trainer drives them — the
    CUDA kernels sit behind forward()/loss()/backward().  This is also what runs when the
    unmodified reference Trainer is handed these model classes.
  * fused mode (optimizer sgd, adagrad or adam, config.fused_step not False): the step is issued
    as a few kernels with no autograd graph and no torch optimizer:
      pairwise hinge + SGD : kge_train_pairwise_hinge_sgd (2 kernels)
      sgd / adagrad        : score_fwd -> loss kernel -> score_bwd (+ reg) -> kge_optim_apply_rows
                             (sparse: zero-gradient rows do not move under SGD/Adagrad, and the touched rows
                             share kge_optim_apply_dense's per-element arithmetic, so the result equals the
                             dense step bit for bit)
      adam (the CLI default, common.py:50): ... -> kge_optim_apply_dense per table — dense Adam moves
                             every row every step, so its exact form is one HBM-bound sweep per table
  * data-parallel (torch.distributed world > 1, tables replicated; SURVEY.md 8e row 3): config.dp_mode
      "grads": every rank scores ITS batch shard forward + backward into the dense gradient buffers,
               ONE all-reduce per table sums (hinge) / averages (mean-type losses) them over NVLink, then
               every rank applies the identical dense optimizer step — per-GPU scoring work is B, not world x B;
      "ids"  : ranks all-gather their batch ids (24 KB at B=512) and every rank applies the global batch —
               cheaper than moving gradient tables when the batch is tiny;
      None   : "grads" when a rank's batch touches more floats than the tables hold, else "ids".

The sampler processes, epoch loop, early stopping, checkpointing and export of the
reference Trainer are out of scope here (SURVEY.md §2 rows 7-8); batches are handed in as
host id arrays, which is what Generator yields (pykg2vec/data/generator.py:97,158).
"""
import numpy as np
import torch
import torch.optim as optim

from . import _lib
from .evaluator import Evaluator
from .KGMeta import TrainingStrategy


class Trainer:
    def __init__(self, model, config):
        self.model = model
        self.config = config
        self.evaluator = None
        self.optimizer = None
        self._fused = False
        self._grad_scratch = None
        self._state = None
        self._pinned = None
        self._loss_buf = None
        self._graphs = {}
        self._state2 = None
        self._step = 0
        self._selfadv_fused = True
        self._world = 1
        self._dp = None

    def build_model(self):
        """trainer.py:103-144 (optimizer selection; unknown names raise NotImplementedError)."""
        self.evaluator = Evaluator(self.model, self.config)
        self.model.to(self.config.device)
        name = self.config.optimizer
        lr = self.config.learning_rate
        if name == "adam":
            self.optimizer = optim.Adam(self.model.parameters(), lr=lr)
        elif name == "sgd":
            self.optimizer = optim.SGD(self.model.parameters(), lr=lr)
        elif name == "adagrad":
            self.optimizer = optim.Adagrad(self.model.parameters(), lr=lr)
        elif name == "rms":
            self.optimizer = optim.RMSprop(self.model.parameters(), lr=lr)
        else:
            raise NotImplementedError("No support for %s optimizer" % name)
        self._fused = name in ("sgd", "adagrad", "adam") and getattr(self.config, "fused_step", True) and \
            hasattr(self.model, "kge_desc") and not getattr(self.model, "kge_dense_params", False)
        if self._fused:
            tabs = self.model.kge_tables()
            self._grad_scratch = [torch.zeros_like(t) if t.requires_grad else None for t in tabs]
            if name in ("adagrad", "adam"):  # optim.Adagrad: state_sum = 0; optim.Adam: exp_avg = exp_avg_sq = 0
                self._state = [torch.zeros_like(t) if t.requires_grad else None for t in tabs]
            if name == "adam":
                self._state2 = [torch.zeros_like(t) if t.requires_grad else None for t in tabs]
        self._step = 0
        self._loss_buf = torch.zeros(1, dtype=torch.float32, device=self.config.device)
        import torch.distributed as dist
        self._world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self._dp = None
        if self._world > 1 and self._fused:
            self._dp = getattr(self.config, "dp_mode", None) or self._pick_dp_mode()
            if self._dp == "off":   # every rank trains on its own (tests: the single-process yardstick)
                self._dp = None

    def _pick_dp_mode(self):
        """'grads' (shard the scoring, all-reduce dense gradients) pays when the rows a local batch touches
        outweigh one sweep over the tables; tiny batches exchange ids instead — for plain SGD only.

        Replica consistency decides the rest.  In 'grads' mode every rank applies the SAME all-reduced gradient, so
        the replicas stay bit-identical.  In 'ids' mode every rank accumulates the global batch itself with float
        atomics (unordered): the gradients agree to rounding only.  SGD carries that rounding through unchanged
        (w -= lr g: replicas agree to ~1e-7 relative), but Adagrad and Adam DIVIDE by a gradient magnitude, so an
        element whose contributions cancel to ~0 can step by +-lr in opposite directions on two ranks
        (tests/test_gpu_multi.py saw 1e-3 after three Adam steps) — those optimizers always get 'grads'."""
        if self.config.optimizer != "sgd":
            return "grads"
        tabs = [t for t in self.model.kge_tables() if t.requires_grad]
        table_floats = sum(t.numel() for t in tabs)
        per_triple = sum(t.shape[1] for t in tabs)
        batch = int(self.config.batch_size) * (1 + int(getattr(self.config, "neg_rate", 1)))
        # a rank's own batch already touches more floats than the tables hold -> sweep-sized exchanges are cheap
        # next to the scoring work, and splitting that work is what pays (config 4); below that the 24 KB id
        # exchange (which hides behind an evaluation batch) beats moving gradient tables (config 2)
        return "grads" if batch * per_triple >= table_floats else "ids"

    # ---- reference-signature steps (autograd mode) --------------------------------------------
    def train_step_pairwise(self, pos_h, pos_r, pos_t, neg_h, neg_r, neg_t):
        pos_preds = self.model(pos_h, pos_r, pos_t)
        neg_preds = self.model(neg_h, neg_r, neg_t)
        if self.model.model_name.lower() == "rotate":
            loss = self.model.loss(pos_preds, neg_preds, self.config.neg_rate, self.config.alpha)
        else:
            loss = self.model.loss(pos_preds, neg_preds, self.config.margin)
        loss = loss + self.model.get_reg(None, None, None)
        return loss

    def train_step_pointwise(self, h, r, t, target):
        preds = self.model(h, r, t)
        loss = self.model.loss(preds, target.type(preds.type()))
        loss = loss + self.model.get_reg(h, r, t)
        return loss

    def train_step_projection(self, h, r, t, hr_t, tr_h):
        """trainer.py:159-174: both directions through the model, Criterion.multi_class_bce over the
        dense [b,N] label matrices (ConvE family) or the model's own loss terms (ProjE)."""
        if self.model.model_name.lower() in ["conve", "tucker", "interacte", "hyper", "acre"]:
            pred_tails = self.model(h, r, direction="tail")
            pred_heads = self.model(t, r, direction="head")
            if hasattr(self.config, 'label_smoothing'):
                loss = self.model.loss(pred_heads, pred_tails, tr_h, hr_t, self.config.label_smoothing,
                                       self.config.tot_entity)
            else:
                loss = self.model.loss(pred_heads, pred_tails, tr_h, hr_t, None, None)
        else:
            pred_tails = self.model(h, r, hr_t, direction="tail")
            pred_heads = self.model(t, r, tr_h, direction="head")
            loss = self.model.loss(pred_heads, pred_tails)
        loss = loss + self.model.get_reg(h, r, t)
        return loss

    def _projection_batch(self, data):
        """[h, r, t, hr_t, tr_h] as Generator yields them for PROJECTION_BASED models
        (generator.py:160-230: three id arrays and two dense [b, N] label tensors)."""
        dev = self.config.device
        ids, nbytes = self._to_device(list(data[:3]))
        labels = []
        for lab in data[3:5]:
            lab = torch.as_tensor(lab, dtype=torch.float32)
            if not lab.is_cuda:
                nbytes += lab.numel() * 4
                lab = lab.to(dev, non_blocking=True)
            labels.append(lab)
        return ids + labels, nbytes

    # ---- fused steps --------------------------------------------------------------------------
    def _opt_code(self):
        return {"sgd": _lib.OPT_SGD, "adagrad": _lib.OPT_ADAGRAD, "adam": _lib.OPT_ADAM}[self.config.optimizer]

    def _dense_apply(self, desc, lr):
        """optimizer.step() as one sweep per table over its dense gradient buffer (Adam always; SGD /
        Adagrad after a data-parallel gradient all-reduce, where the touched rows are the union over ranks)."""
        self._step += 1
        state2 = self._state2
        for k, w in enumerate(desc.tables):
            g = self._grad_scratch[k]
            if g is None:
                continue
            _lib.optim_apply_dense(w, g, self._opt_code(), lr, self._state[k] if self._state else None,
                                   state2[k] if state2 else None, step=self._step)

    def _apply(self, desc, id_sets, lr):
        if self.config.optimizer == "adam" or self._dp == "grads":
            return self._dense_apply(desc, lr)
        for h, r, t in id_sets:
            _lib.optim_apply_rows(desc, self._grad_scratch, self._state, self._opt_code(), h, r, t, lr)

    def _allreduce_grads(self, loss, mean_type):
        """data-parallel 'grads' mode: ONE NCCL all-reduce per gradient table (sum for the hinge's sum over
        pairs, average for the mean-type losses and regularisers) + the scalar loss."""
        if self._dp != "grads":
            return loss
        import torch.distributed as dist
        native_avg = mean_type and dist.get_backend() == "nccl"   # gloo has no AVG: sum, then scale
        op = dist.ReduceOp.AVG if native_avg else dist.ReduceOp.SUM
        bufs = [g for g in self._grad_scratch if g is not None] + [loss]
        for b in bufs:
            dist.all_reduce(b, op=op)
            if mean_type and not native_avg:
                b.div_(self._world)
        return loss

    def _fused_pairwise(self, ids):
        self.model.kge_pre_score()   # Rescal: in-place row normalisation, as its forward() does
        desc = self.model.kge_desc()
        ph, pr, pt, nh, nr, nt = ids
        lr = float(self.config.learning_rate)
        rotate = self.model.model_name.lower() == "rotate"
        if not rotate and nh.numel() != ph.numel():
            # Criterion.pairwise_hinge subtracts pos [B] and neg [B*neg_rate] elementwise: the reference
            # raises a broadcast error for neg_rate > 1 (criterion.py:26-29) — so does this path
            raise ValueError("pairwise hinge needs one negative per positive (got %d positives, %d negatives)"
                             % (ph.numel(), nh.numel()))
        if not rotate and self.config.optimizer == "sgd" and self._dp != "grads":
            _lib.train_pairwise_hinge_sgd(desc, self._grad_scratch, ph, pr, pt, nh, nr, nt,
                                          float(self.config.margin), lr, self._loss_buf)
            return self._loss_buf
        loss = None
        if rotate and self._selfadv_fused:
            # forward (positives + negatives) + self-adversarial loss + backward in ONE kernel
            try:
                loss = _lib.train_pairwise_selfadv(desc, self._grad_scratch, ph, pr, pt, nh, nr, nt,
                                                   int(self.config.neg_rate), float(self.config.alpha))
            except _lib.KgeNotSupported:   # neg_rate beyond a CTA's shared memory: the five-launch path
                self._selfadv_fused = False
        if loss is None:
            pos = _lib.score_fwd(desc, ph, pr, pt)
            neg = _lib.score_fwd(desc, nh, nr, nt)
            if rotate:
                loss, gp, gn = _lib.loss_selfadv(pos, neg, int(self.config.neg_rate), float(self.config.alpha))
            else:
                loss, gp, gn = _lib.loss_pairwise_hinge(pos, neg, float(self.config.margin))
            _lib.score_bwd(desc, ph, pr, pt, gp, self._grad_scratch)
            _lib.score_bwd(desc, nh, nr, nt, gn, self._grad_scratch)
        loss = self._allreduce_grads(loss, mean_type=rotate)
        self._apply(desc, ((ph, pr, pt), (nh, nr, nt)), lr)
        return loss

    def _fused_pointwise(self, ids):
        self.model.kge_pre_score()
        desc = self.model.kge_desc()
        h, r, t, y = ids
        lr = float(self.config.learning_rate)
        if y.dtype == torch.int64 and y.is_contiguous():   # forward + logistic loss + backward in ONE kernel
            loss = _lib.train_pointwise_logistic(desc, self._grad_scratch, h, r, t, y)
        else:
            preds = _lib.score_fwd(desc, h, r, t)
            loss, g = _lib.loss_pointwise_logistic(preds, y.to(torch.float32))
            _lib.score_bwd(desc, h, r, t, g, self._grad_scratch)
        hook = self.model.kge_fused_reg()
        if hook is not None:
            reg = _lib.reg_fwd_bwd(desc, hook[0], hook[1], h, r, t, grad_scale=1.0, grad_tables=self._grad_scratch)
        else:   # SimplE / SimplE_ignr: get_reg acts on the id tensors — a constant w.r.t. the weights
            reg = self.model.get_reg(h, r, t).detach().to(torch.float32).reshape(1)
        loss = self._allreduce_grads(loss + reg, mean_type=True)
        self._apply(desc, ((h, r, t),), lr)
        return loss

    # ---- one batch, host ids in, host loss out (trainer.py:269-300) -----------------------------
    def _to_device(self, arrays):
        """Pack the batch's id arrays into one pinned staging buffer and issue ONE H2D copy
        (the reference issues one pageable copy per array, trainer.py:288-293)."""
        k = len(arrays)
        n = max(len(a) for a in arrays)
        if self._pinned is None or self._pinned.shape[0] < k or self._pinned.shape[1] < n:
            self._pinned = torch.empty((k, n), dtype=torch.int64).pin_memory()
        lens = []
        for i, a in enumerate(arrays):
            a = np.asarray(a, dtype=np.int64)
            self._pinned[i, :len(a)] = torch.from_numpy(a)
            lens.append(len(a))
        dev = self._pinned[:k, :n].to(self.config.device, non_blocking=True)
        return [dev[i, :lens[i]] for i in range(k)], k * n * 8

    def _graphed_hinge_step(self, data, sync=True):
        """Pairwise hinge + SGD as ONE CUDA graph: H2D of the packed [6,B] ids from a pinned
        buffer, the two training kernels, D2H of the loss.  Data parallel in "ids" mode: the H2D copy and the
        NCCL all-gather of the ids are issued eagerly, the graph holds the step on the gathered global batch."""
        from .graphs import StagedGraph
        B = len(data[0])
        tables = self.model.kge_tables()
        key = (B, tuple(int(w.data_ptr()) for w in tables))
        call = self._graphs.get(key)
        if call is None:
            desc = self.model.kge_desc()
            loss = torch.zeros(1, dtype=torch.float32, device=self.config.device)
            margin, lr = float(self.config.margin), float(self.config.learning_rate)
            world = self._world if self._dp == "ids" else 1
            gath = torch.zeros((world * 6, B), dtype=torch.int64, device=self.config.device) if world > 1 else None

            def make_body(step_lr):
                def body(d_in):
                    if world > 1:   # rank-major gathered blocks -> [6, world * B]
                        ids = gath.view(world, 6, B).permute(1, 0, 2).reshape(6, world * B).contiguous()
                    else:
                        ids = d_in.view(6, B)
                    self.model.kge_pre_score()   # captured with the step (Rescal's in-place normalisation)
                    _lib.train_pairwise_hinge_sgd(desc, self._grad_scratch, ids[0], ids[1], ids[2], ids[3],
                                                  ids[4], ids[5], margin, step_lr, loss)
                    return loss
                return body

            pre = None
            if world > 1:
                import torch.distributed as dist

                def pre(d_in):
                    dist.all_gather_into_tensor(gath, d_in.view(6, B))

            # the warm-up run before capture uses lr = 0: the tables are left exactly unchanged
            call = StagedGraph(self.config.device, 6 * B, torch.empty(1, dtype=torch.float32), make_body(lr),
                               warm_body=make_body(0.0), pre=pre,
                               capture_error_mode="thread_local" if world > 1 else "global").capture()
            self._graphs[key] = call
        call.wait_idle()  # an earlier asynchronous step may still be reading the staging buffer
        buf = call.h_in.numpy().reshape(6, B)
        for i, a in enumerate(data):
            buf[i] = a
        self.last_h2d_bytes = 6 * B * 8
        if not sync:
            from .graphs import PendingScalar
            call(sync=False)
            return PendingScalar(call)
        return float(call()[0])

    def exchange_batch_async(self, ids):
        """data-parallel "ids" mode: start the all-gather of this rank's batch ids (NCCL runs it on its own
        stream) and return a closure yielding the global batch — issue it BEFORE independent work (an
        evaluation batch) and hand the closure to train_batch_device(exchanged=...) so that the exchange hides
        behind that work.  None in every other mode."""
        if self._dp != "ids":
            return None
        from . import sharding
        ids = list(ids)
        n = [int(a.numel()) for a in ids]
        if len(set(n)) == 1:
            fin = sharding.allgather_batch_ids_async(torch.stack(ids))
            return lambda: list(fin())
        k = len(ids) // 2   # ragged (neg_rate > 1): positives and negatives gathered separately
        fa = sharding.allgather_batch_ids_async(torch.stack(ids[:k]))
        fb = sharding.allgather_batch_ids_async(torch.stack(ids[k:]))
        return lambda: list(fa()) + list(fb())

    def train_batch_device(self, ids, exchanged=None):
        """One batch whose id arrays are already DEVICE tensors (pykg2vec_b200.generator.Generator).
        Returns the loss as a device tensor (no host sync)."""
        self.model.train()
        ids = list(ids)
        strategy = self.model.training_strategy
        if self._dp == "ids":   # replicated update on the all-gathered global batch
            ids = (exchanged or self.exchange_batch_async(ids))()
        if self._fused:
            with torch.no_grad():
                if strategy == TrainingStrategy.PAIRWISE_BASED:
                    return self._fused_pairwise(ids)
                if strategy == TrainingStrategy.POINTWISE_BASED:
                    return self._fused_pointwise(ids)
                raise NotImplementedError("Unknown training strategy: %s" % strategy)
        self.optimizer.zero_grad()
        if strategy == TrainingStrategy.PAIRWISE_BASED:
            loss = self.train_step_pairwise(*ids)
        elif strategy == TrainingStrategy.POINTWISE_BASED:
            loss = self.train_step_pointwise(*ids)
        elif strategy == TrainingStrategy.PROJECTION_BASED:
            loss = self.train_step_projection(*ids)
        else:
            raise NotImplementedError("Unknown training strategy: %s" % strategy)
        loss.backward()
        self.optimizer.step()
        return loss.detach()

    def train_model_epoch(self, generator, num_batch=None):
        """Trainer.train_model_epoch (trainer.py:259-307) over a device-side Generator: the
        accumulated loss stays on the device until the end of the epoch (one sync per epoch
        instead of one `loss.item()` per batch, trainer.py:300)."""
        if num_batch is None:
            num_batch = self.config.tot_train_triples // self.config.batch_size
        generator.start_one_epoch(num_batch)
        acc = torch.zeros((), dtype=torch.float32, device=self.config.device)
        for _ in range(num_batch):
            acc += self.train_batch_device(next(generator)).reshape(())
        return float(acc.item())

    def train_batch(self, data, sync=True):
        """data: the list Generator yields — 6 id arrays (pairwise) or 4 (pointwise).  Returns the
        batch loss as a float (the reference reads `loss.item()` per batch, trainer.py:300).
        sync=False (graph-staged steps only) returns a handle instead — float(handle) waits for the
        D2H copy — so the caller's next host work overlaps this step's kernels."""
        self.model.train()
        data = list(data)
        if (self._fused and getattr(self.config, "cuda_graph", True) and self._dp in (None, "ids")
                and self.model.training_strategy == TrainingStrategy.PAIRWISE_BASED
                and self.model.model_name.lower() != "rotate" and self.config.optimizer == "sgd"
                and len(data) == 6 and all(len(a) == len(data[0]) for a in data)):
            return self._graphed_hinge_step(data, sync=sync)
        strategy = self.model.training_strategy
        if strategy == TrainingStrategy.PROJECTION_BASED:
            ids, nbytes = self._projection_batch(data)
        else:
            ids, nbytes = self._to_device(list(data))
        self.last_h2d_bytes = nbytes
        if self._fused:
            loss = self.train_batch_device(ids)
            if not sync:
                return loss                # device tensor; float(loss) syncs when the caller wants the value
            return float(loss.item())  # D2H sync, as acc_loss += loss.item() (trainer.py:300)
        self.optimizer.zero_grad()
        if strategy == TrainingStrategy.PAIRWISE_BASED:
            loss = self.train_step_pairwise(*ids)
        elif strategy == TrainingStrategy.POINTWISE_BASED:
            loss = self.train_step_pointwise(*ids)
        elif strategy == TrainingStrategy.PROJECTION_BASED:
            loss = self.train_step_projection(*ids)
        else:
            raise NotImplementedError("Unknown training strategy: %s" % strategy)
        loss.backward()
        self.optimizer.step()
        return float(loss.item())
