"""Evaluator / MetricCalculator — mirror of pykg2vec/utils/evaluator.py.

Same constructor, `test_tail_rank / test_head_rank / test_rel_rank`, `mini_test`,
`full_test`, `test` entry points and the same MetricCalculator metric dictionaries, but
`test()` no longer walks one triple at a time (evaluator.py:313-326: two forwards over
all N entities, a full topk sort, a D2H copy of N ids and a Python loop per triple):
queries are ranked in batches by the 1-vs-all counting kernel (kge_rank_1vsall) and only
Q x 4 int32 ranks come back to the host.
"""
import os
import timeit

import numpy as np
import torch

from . import _lib


class MetricCalculator:
    """Mirror of evaluator.py:14-230 (metric bookkeeping is host logic and stays Python)."""

    def __init__(self, config):
        self.config = config
        self.hr_t = config.knowledge_graph.read_cache_data('hr_t')
        self.tr_h = config.knowledge_graph.read_cache_data('tr_h')
        self.mr, self.fmr, self.mrr, self.fmrr, self.hit, self.fhit = {}, {}, {}, {}, {}, {}
        self.epoch = None
        self.reset()

    def reset(self):
        self.rank_head, self.rank_tail, self.f_rank_head, self.f_rank_tail = [], [], [], []
        self.epoch = None
        self.start_time = timeit.default_timer()

    # -- reference-compatible slow path: sorted candidate lists (evaluator.py:54-123) --------
    def append_result(self, result):
        predict_tail, predict_head = result[0], result[1]
        h, r, t = result[2], result[3], result[4]
        self.epoch = result[5]
        t_rank, f_t_rank = self.get_tail_rank(predict_tail, h, r, t)
        h_rank, f_h_rank = self.get_head_rank(predict_head, h, r, t)
        self.rank_head.append(h_rank)
        self.rank_tail.append(t_rank)
        self.f_rank_head.append(f_h_rank)
        self.f_rank_tail.append(f_t_rank)

    def get_tail_rank(self, tail_candidate, h, r, t):
        trank = ftrank = 0
        known = self.hr_t[(h, r)]
        for j in range(len(tail_candidate)):
            val = tail_candidate[-j - 1]
            if val == t:
                break
            trank += 1
            ftrank += 1
            if val in known:
                ftrank -= 1
        return trank, ftrank

    def get_head_rank(self, head_candidate, h, r, t):
        hrank = fhrank = 0
        known = self.tr_h[(t, r)]
        for j in range(len(head_candidate)):
            val = head_candidate[-j - 1]
            if val == h:
                break
            hrank += 1
            fhrank += 1
            if val in known:
                fhrank -= 1
        return hrank, fhrank

    # -- fast path: ranks counted on the device ---------------------------------------------
    def append_ranks(self, counts, epoch):
        """counts: [Q,4] int array of 0-based (trank, ftrank, hrank, fhrank)."""
        c = np.asarray(counts)
        self.epoch = epoch
        self.rank_tail.extend(c[:, 0].tolist())
        self.f_rank_tail.extend(c[:, 1].tolist())
        self.rank_head.extend(c[:, 2].tolist())
        self.f_rank_head.extend(c[:, 3].tolist())

    def settle(self):
        """evaluator.py:125-141."""
        head_ranks = np.asarray(self.rank_head, dtype=np.float32) + 1
        tail_ranks = np.asarray(self.rank_tail, dtype=np.float32) + 1
        head_franks = np.asarray(self.f_rank_head, dtype=np.float32) + 1
        tail_franks = np.asarray(self.f_rank_tail, dtype=np.float32) + 1
        ranks = np.concatenate((head_ranks, tail_ranks))
        franks = np.concatenate((head_franks, tail_franks))
        self.mr[self.epoch] = np.mean(ranks)
        self.mrr[self.epoch] = np.mean(np.reciprocal(ranks))
        self.fmr[self.epoch] = np.mean(franks)
        self.fmrr[self.epoch] = np.mean(np.reciprocal(franks))
        for hit in self.config.hits:
            self.hit[(self.epoch, hit)] = np.mean(ranks <= hit, dtype=np.float32)
            self.fhit[(self.epoch, hit)] = np.mean(franks <= hit, dtype=np.float32)

    def get_curr_scores(self):
        return {'mr': self.mr[self.epoch], 'fmr': self.fmr[self.epoch],
                'mrr': self.mrr[self.epoch], 'fmrr': self.fmrr[self.epoch]}

    def display_summary(self):
        stop_time = timeit.default_timer()
        lines = ['', "------Test Results for %s: Epoch: %s --- time: %.2f------------"
                 % (getattr(self.config, 'dataset_name', '?'), str(self.epoch), stop_time - self.start_time),
                 '--# of entities, # of relations: %d, %d' % (self.config.tot_entity, self.config.tot_relation),
                 '--mr,  filtered mr             : %.4f, %.4f' % (self.mr[self.epoch], self.fmr[self.epoch]),
                 '--mrr, filtered mrr            : %.4f, %.4f' % (self.mrr[self.epoch], self.fmrr[self.epoch])]
        for hit in self.config.hits:
            lines.append('--hits%d                        : %.4f ' % (hit, self.hit[(self.epoch, hit)]))
            lines.append('--filtered hits%d               : %.4f ' % (hit, self.fhit[(self.epoch, hit)]))
        lines += ["---------------------------------------------------------", '']
        if getattr(self.config, 'verbose', False):
            print("\n".join(lines))
        return "\n".join(lines)


def build_filter_csr(keys, dct):
    """CSR (ptr[Q+1], idx[nnz]) int64 numpy of the known-positive sets dct[key] per query."""
    ptr = np.zeros(len(keys) + 1, dtype=np.int64)
    chunks = []
    for i, k in enumerate(keys):
        s = dct.get(k, ())
        ptr[i + 1] = ptr[i] + len(s)
        if len(s):
            chunks.append(np.fromiter(s, dtype=np.int64, count=len(s)))
    idx = np.concatenate(chunks) if chunks else np.zeros(0, dtype=np.int64)
    return ptr, idx


class Evaluator:
    """Mirror of evaluator.py:233-334."""

    QUERY_BATCH = 8192  # queries per kge_rank_1vsall call (<= 65535)

    def __init__(self, model, config, tuning=False):
        self.model = model
        self.config = config
        self.tuning = tuning
        self.test_data = self.config.knowledge_graph.read_cache_data('triplets_test')
        self.eval_data = self.config.knowledge_graph.read_cache_data('triplets_valid')
        self.metric_calculator = MetricCalculator(self.config)
        self._workspace = None
        self._filter_cache = {}

    # ---- single-query API used by Trainer.infer_* (trainer.py:330-386) ---------------------
    def _dev(self):
        return torch.device(self.config.device)

    def test_tail_rank(self, h, r, topk=-1):
        """ids in DESCENDING score order, length topk (evaluator.py:249-260; worst first for
        distance models — the caller reads the list from its end)."""
        if hasattr(self.model, 'predict_tail_rank'):
            return self.model.predict_tail_rank(torch.LongTensor([h]).to(self._dev()),
                                                torch.LongTensor([r]).to(self._dev()), topk=topk).squeeze(0)
        n = self.config.tot_entity
        dev = self._dev()
        h_batch = torch.full((n,), int(h), dtype=torch.long, device=dev)
        r_batch = torch.full((n,), int(r), dtype=torch.long, device=dev)
        entity_array = torch.arange(n, dtype=torch.long, device=dev)
        preds = self.model.forward(h_batch, r_batch, entity_array)
        _, rank = torch.topk(preds, k=topk)
        return rank

    def test_head_rank(self, r, t, topk=-1):
        if hasattr(self.model, 'predict_head_rank'):
            return self.model.predict_head_rank(torch.LongTensor([t]).to(self._dev()),
                                                torch.LongTensor([r]).to(self._dev()), topk=topk).squeeze(0)
        n = self.config.tot_entity
        dev = self._dev()
        entity_array = torch.arange(n, dtype=torch.long, device=dev)
        r_batch = torch.full((n,), int(r), dtype=torch.long, device=dev)
        t_batch = torch.full((n,), int(t), dtype=torch.long, device=dev)
        preds = self.model.forward(entity_array, r_batch, t_batch)
        _, rank = torch.topk(preds, k=topk)
        return rank

    def test_rel_rank(self, h, t, topk=-1):
        if hasattr(self.model, 'predict_rel_rank'):
            return self.model.predict_rel_rank(h.to(self._dev()), t.to(self._dev()), topk=topk).squeeze(0)
        n = self.config.tot_relation
        dev = self._dev()
        h_batch = torch.full((n,), int(h), dtype=torch.long, device=dev)
        rel_array = torch.arange(n, dtype=torch.long, device=dev)
        t_batch = torch.full((n,), int(t), dtype=torch.long, device=dev)
        preds = self.model.forward(h_batch, rel_array, t_batch)
        _, rank = torch.topk(preds, k=topk)
        return rank

    # ---- batched ranking ---------------------------------------------------------------------
    def rank_triples(self, hs, rs, ts, filt_t=None, filt_h=None):
        """0-based (trank, ftrank, hrank, fhrank) for host id arrays -> numpy int32 [Q,4].
        Host buffers in, host ranks out: this is the end-to-end call bench.py times.
        Per batch of <= QUERY_BATCH queries: ids and filter CSRs are packed into one pinned
        buffer (one H2D copy), the rank kernels run, and the [q,4] counts come back in one D2H
        copy; the whole round trip is a CUDA graph keyed on the batch geometry."""
        hs = np.ascontiguousarray(hs, dtype=np.int64)
        rs = np.ascontiguousarray(rs, dtype=np.int64)
        ts = np.ascontiguousarray(ts, dtype=np.int64)
        Q = hs.shape[0]
        out = np.empty((Q, 4), dtype=np.int32)
        self.last_h2d_bytes = 0
        self.last_d2h_bytes = 0
        if hasattr(self.model, "proj_query"):
            return self._rank_triples_projection(hs, rs, ts, filt_t, filt_h, out)
        if self._use_relation_groups(rs):
            return self._rank_triples_by_relation(hs, rs, ts, filt_t, filt_h, out)
        for lo in range(0, Q, self.QUERY_BATCH):
            hi = min(Q, lo + self.QUERY_BATCH)
            q = hi - lo
            if filt_t is not None:
                tp, ti = filt_t
                hp, hidx = filt_h
                tptr, tidx = tp[lo:hi + 1] - tp[lo], ti[tp[lo]:tp[hi]]
                hptr, hix = hp[lo:hi + 1] - hp[lo], hidx[hp[lo]:hp[hi]]
            else:
                tptr = hptr = np.zeros(q + 1, dtype=np.int64)
                tidx = hix = np.zeros(0, dtype=np.int64)
            call = self._rank_call(q, len(tidx), len(hix))
            buf = call.h_in.numpy()
            o = 0
            for a in (hs[lo:hi], rs[lo:hi], ts[lo:hi], tptr, hptr):
                buf[o:o + len(a)] = a
                o += len(a)
            buf[o:o + len(tidx)] = tidx
            o2 = o + call.cap_t
            buf[o2:o2 + len(hix)] = hix
            res = call()
            out[lo:hi] = res.numpy()
            self.last_h2d_bytes += call.h_in.numel() * 8
            self.last_d2h_bytes += res.numel() * 4
        return out

    # ---- TransH / TransD: relation-grouped evaluation ---------------------------------------------
    GROUP_MIN_QUERIES_PER_RELATION = 32
    GROUPED_BY_DEFAULT = None    # None: decide by queries per distinct relation (bench_grouped.py times both paths)

    def _use_relation_groups(self, rs):
        """TransH / TransD project the candidate rows with a relation-dependent vector, so their
        1-vs-all sweep is the per-pair gather kernel (every pair re-reads and re-projects the
        candidate row).  When a batch holds many test triples per relation it is cheaper to project
        the whole entity table once per relation (kge_project_entities) and rank that relation's
        queries with TransE's tiled sweep over the projected table — same bits, hence same ranks
        (tests/test_emu_project.py, tests/test_gpu_score_rank.py).  FB15k-237 shape, 20,466 test
        triples: TransH 349 -> 30 ms, TransD 344 -> 111 ms, identical ranks.  config.relation_grouped_eval:
        True / False forces the choice, None (default) decides by queries per distinct relation."""
        name = getattr(self.model, "model_name", "")
        if len(rs) == 0:
            return False
        if name not in ("transh", "transd", "transr"):   # TransR: P_r = normalize(ent) . M_r over once-normalised rel rows
            return False
        force = getattr(self.config, "relation_grouped_eval", self.GROUPED_BY_DEFAULT)
        if force is not None:
            return bool(force)
        return len(rs) >= self.GROUP_MIN_QUERIES_PER_RELATION * len(np.unique(rs))

    def _rank_triples_by_relation(self, hs, rs, ts, filt_t, filt_h, out):
        dev = self._dev()
        Q = hs.shape[0]
        order = np.argsort(rs, kind="stable")
        rel_sorted = rs[order]
        starts = np.flatnonzero(np.r_[True, rel_sorted[1:] != rel_sorted[:-1]])
        ends = np.r_[starts[1:], Q]

        def reorder(filt):   # CSR rows permuted into the sorted query order
            if filt is None:
                return None
            ptr, idx = np.asarray(filt[0], dtype=np.int64), np.asarray(filt[1], dtype=np.int64)
            lens = (ptr[1:] - ptr[:-1])[order]
            new_ptr = np.zeros(Q + 1, dtype=np.int64)
            np.cumsum(lens, out=new_ptr[1:])
            take = np.repeat(ptr[:-1][order] - new_ptr[:-1], lens) + np.arange(new_ptr[-1], dtype=np.int64)
            return new_ptr, idx[take]

        ft, fh = reorder(filt_t), reorder(filt_h)
        parts = [hs[order], rel_sorted, ts[order]]
        if ft is not None:
            parts += [ft[0], fh[0], ft[1], fh[1]]
        words = sum(len(a) for a in parts)
        stage = torch.empty(words, dtype=torch.int64).pin_memory()
        buf, o, v = stage.numpy(), 0, []
        for a in parts:
            buf[o:o + len(a)] = a
            v.append((o, o + len(a)))
            o += len(a)
        d_in = stage.to(dev, non_blocking=True)
        v = [d_in[a:b] for a, b in v]
        desc = self.model.kge_desc()
        if desc.name == "transr":   # TransE of width rel_dim over [normalize(ent) . M_r, normalize(rel)]
            width, rel_rows = desc.rel_dim, _lib.normalize_rows_to(desc.tables[1])
        else:
            width, rel_rows = desc.dim, desc.tables[1]
        proj = torch.empty((desc.num_ent, width), dtype=torch.float32, device=dev)
        te = _lib.ModelDesc("transe", [proj, rel_rows], width, l1_flag=desc.l1_flag)
        counts = torch.zeros((Q, 4), dtype=torch.int32, device=dev)
        ws = torch.empty(max(_lib.rank_workspace_bytes(te, min(Q, 65535)), 16), dtype=torch.uint8, device=dev)
        for a, b in zip(starts.tolist(), ends.tolist()):
            _lib.project_entities(desc, int(rel_sorted[a]), proj)
            for lo in range(a, b, 65535):
                hi = min(b, lo + 65535)
                f_t = f_h = None
                if ft is not None:
                    tp, hp = v[3][lo:hi + 1], v[4][lo:hi + 1]
                    f_t = ((tp - tp[0]).contiguous(), v[5][int(ft[0][lo]):int(ft[0][hi])])
                    f_h = ((hp - hp[0]).contiguous(), v[6][int(fh[0][lo]):int(fh[0][hi])])
                    if f_t[1].numel() == 0:
                        f_t = None
                    if f_h[1].numel() == 0:
                        f_h = None
                _lib.rank_1vsall(te, v[0][lo:hi], v[1][lo:hi], v[2][lo:hi], f_t, f_h, counts=counts[lo:hi],
                                 workspace=ws)
        out[order] = counts.cpu().numpy()
        self.last_h2d_bytes = words * 8
        self.last_d2h_bytes = Q * 16
        return out

    def _rank_triples_projection(self, hs, rs, ts, filt_t, filt_h, out):
        """Projection models (ConvE, ...): the reference evaluates them one query at a time through
        predict_tail_rank / predict_head_rank — a [1,N] forward plus a full topk each
        (evaluator.py:249-263, projection.py:119-125).  Here a batch of queries goes through the
        model's trunk once per direction and kge_proj_rank counts the better-scored entities
        without materialising [Q,N] predictions."""
        dev = self._dev()
        Q = hs.shape[0]
        ent, bias = self.model.proj_tail_tables()
        # TuckER: the core matrices of the relations present, built once for every batch and both directions of
        # this call (never kept longer: a training step may rewrite the weights behind torch's back)
        make_cores = getattr(self.model, "proj_query_cores", None)
        cores = make_cores(torch.from_numpy(np.unique(rs)).to(dev)) if make_cores is not None and Q else None
        kw = {"cores": cores} if cores is not None else {}
        for lo in range(0, Q, self.QUERY_BATCH):
            hi = min(Q, lo + self.QUERY_BATCH)
            q = hi - lo
            parts = [hs[lo:hi], rs[lo:hi], ts[lo:hi]]
            if filt_t is not None:
                tp, ti = filt_t
                hp, hidx = filt_h
                parts += [tp[lo:hi + 1] - tp[lo], hp[lo:hi + 1] - hp[lo], ti[tp[lo]:tp[hi]], hidx[hp[lo]:hp[hi]]]
            words = sum(len(a) for a in parts)
            stage = getattr(self, "_proj_stage", None)
            if stage is None or stage.numel() < words:   # pinned staging buffer, grown geometrically
                stage = self._proj_stage = torch.empty(max(words, 2 * (stage.numel() if stage is not None else 0)),
                                                       dtype=torch.int64).pin_memory()
            stage = stage[:words]
            buf, o, views = stage.numpy(), 0, []
            for a in parts:
                buf[o:o + len(a)] = a
                views.append((o, o + len(a)))
                o += len(a)
            d_in = stage.to(dev, non_blocking=True)
            v = [d_in[a:b] for a, b in views]
            h, r, t = v[0], v[1], v[2]
            ft = (v[3], v[5]) if filt_t is not None and len(parts[5]) else None
            fh = (v[4], v[6]) if filt_t is not None and len(parts[6]) else None
            counts = torch.zeros((q, 4), dtype=torch.int32, device=dev)
            x_t = self.model.proj_query(h, r, direction="tail", **kw).contiguous()
            x_h = self.model.proj_query(t, r, direction="head", **kw).contiguous()
            bias_row = bias.detach() if bias is not None else None
            _lib.proj_rank(x_t, ent.detach(), bias_row, t, ft, 0, counts)
            _lib.proj_rank(x_h, ent.detach(), bias_row, h, fh, 1, counts)
            out[lo:hi] = counts.cpu().numpy()
            self.last_h2d_bytes += words * 8
            self.last_d2h_bytes += q * 16
        return out

    @staticmethod
    def _bucket(n):
        cap = 256
        while cap < n:
            cap *= 2
        return cap

    def _rank_call(self, q, nnz_t, nnz_h):
        """Graph-captured (H2D, kge_rank_1vsall, D2H) for q queries and filter capacities rounded
        up to powers of two (the kernels read the true entry counts from ptr[q] on the device)."""
        from .graphs import StagedGraph
        dev = self._dev()
        cap_t, cap_h = self._bucket(nnz_t), self._bucket(nnz_h)
        # Models with derived tables (ConvKB's collapsed A, c0 are fresh temporaries of every kge_tables()
        # call) are keyed on their persistent parameters only and re-derive the tables on every call
        # (eager body, no captured pointers); everything else is keyed on the live table pointers.
        dense = bool(getattr(self.model, "kge_dense_params", False))
        if dense:
            ptrs = tuple(int(p_.data_ptr()) for p_ in self.model.parameters())
        else:
            ptrs = tuple(int(w.data_ptr()) for w in self.model.kge_tables())
        key = (q, cap_t, cap_h, dense, ptrs)
        call = self._filter_cache.get(("graph",) + key)
        if call is not None:
            return call
        desc = self.model.kge_desc()
        counts = torch.zeros((q, 4), dtype=torch.int32, device=dev)
        ws = torch.empty(max(_lib.rank_workspace_bytes(desc, q), 16), dtype=torch.uint8, device=dev)
        words = 3 * q + 2 * (q + 1) + cap_t + cap_h
        model = self.model

        def body(d_in):
            o = 3 * q
            qh, qr, qt = d_in[0:q], d_in[q:2 * q], d_in[2 * q:3 * q]
            tptr, hptr = d_in[o:o + q + 1], d_in[o + q + 1:o + 2 * q + 2]
            o += 2 * q + 2
            tidx, hidx = d_in[o:o + cap_t], d_in[o + cap_t:o + cap_t + cap_h]
            counts.zero_()
            if not dense and hasattr(model, "kge_pre_score"):
                model.kge_pre_score()   # Rescal: tables row-normalised in place, as the reference's forward() does
            d = model.kge_desc() if dense else desc
            _lib.rank_1vsall(d, qh, qr, qt, (tptr, tidx), (hptr, hidx), counts=counts, workspace=ws)
            return counts

        call = StagedGraph(dev, words, torch.empty((q, 4), dtype=torch.int32), body)
        call.cap_t, call.cap_h = cap_t, cap_h
        use_graph = getattr(self.config, "cuda_graph", True) and not dense
        if use_graph:
            call.capture()
        else:
            def eager():
                call._run_eager()
                torch.cuda.current_stream(dev).synchronize()
                return call.h_out
            call.__class__ = type("EagerStaged", (StagedGraph,), {"__call__": lambda self_: eager()})
        self._filter_cache[("graph",) + key] = call
        return call

    def _filters_for(self, data, num):
        key = (id(data), num)
        if key not in self._filter_cache:
            mc = self.metric_calculator
            tr = [(data[i].h, data[i].r, data[i].t) for i in range(num)]
            ft = build_filter_csr([(h, r) for h, r, t in tr], mc.hr_t)
            fh = build_filter_csr([(t, r) for h, r, t in tr], mc.tr_h)
            arr = np.asarray(tr, dtype=np.int64).reshape(-1, 3)
            self._filter_cache[key] = (arr, ft, fh)
        return self._filter_cache[key]

    def mini_test(self, epoch=None):
        if self.config.test_num == 0:
            tot_valid_to_test = len(self.eval_data)
        else:
            tot_valid_to_test = min(self.config.test_num, len(self.eval_data))
        if getattr(self.config, 'debug', False):
            tot_valid_to_test = 10
        return self.test(self.eval_data, tot_valid_to_test, epoch=epoch)

    def full_test(self, epoch=None):
        tot_valid_to_test = len(self.test_data)
        if getattr(self.config, 'debug', False):
            tot_valid_to_test = 10
        return self.test(self.test_data, tot_valid_to_test, epoch=epoch)

    def test(self, data, num_of_test, epoch=None):
        self.metric_calculator.reset()
        arr, ft, fh = self._filters_for(data, num_of_test)
        with torch.no_grad():
            counts = self.rank_triples(arr[:, 0], arr[:, 1], arr[:, 2], ft, fh)
        self.metric_calculator.append_ranks(counts, epoch)
        self.metric_calculator.settle()
        self.metric_calculator.display_summary()
        # (the reference also writes a summary txt / csv at the last epoch, evaluator.py:151-206,331-332: result
        #  files are control plane, out of scope — SURVEY.md §2)
        return self.metric_calculator.get_curr_scores()
