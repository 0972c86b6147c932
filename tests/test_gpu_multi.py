"""-m gpu tests that need >= 2 GPUs (skipped otherwise): NCCL path of the sharded evaluation.
With two GPUs visible:  python -m pytest tests/test_gpu_multi.py -m gpu"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, tmp):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    sys.path.insert(0, here)
    import torch.distributed as dist
    import gpu_util as gpu
    import oracle
    from pykg2vec_b200 import sharding
    torch.cuda.set_device(rank)
    sharding.init_distributed(backend="nccl")
    dev = torch.device("cuda", rank)
    # ComplEx, YAGO3-10-like proportions scaled down: entity rows partitioned across the ranks
    N, R, d, Q = 3001, 7, 100, 33
    om, tabs = gpu.synthetic_case("complex", N, R, d, seed=17)
    rng = np.random.RandomState(5)
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt)
    want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
    lo, hi = sharding.shard_range(N, world, rank)
    ent_local = [torch.from_numpy(tabs[0][lo:hi].copy()).to(dev), torch.from_numpy(tabs[1][lo:hi].copy()).to(dev)]
    rel = [torch.from_numpy(tabs[2]).to(dev), torch.from_numpy(tabs[3]).to(dev)]
    ranker = sharding.RowShardedRanker(sharding.cuda_count_fn("complex", d), N, ent_local, rel, (0, 1), (2, 3))
    got = ranker.rank_queries(qh, qr, qt, ft, fh)
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    # replicated tables, sharded queries, one gather of the ranks
    from pykg2vec_b200 import _lib
    full = [torch.from_numpy(t).to(dev) for t in tabs]
    desc = _lib.ModelDesc("complex", full, d)
    qlo, qhi = sharding.shard_range(Q, world, rank)
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    sub = lambda f: (to(f[0][qlo:qhi + 1] - f[0][qlo]), to(f[1][f[0][qlo]:f[0][qhi]]))
    local = _lib.rank_1vsall(desc, to(qh[qlo:qhi]), to(qr[qlo:qhi]), to(qt[qlo:qhi]), sub(ft), sub(fh))
    allr = sharding.gather_query_shards(local, Q)
    np.testing.assert_array_equal(allr.cpu().numpy(), want)
    g = sharding.allgather_batch_ids(torch.full((6, 4), rank, dtype=torch.int64, device=dev))
    assert g[0].tolist() == [0] * 4 + [1] * 4
    dist.barrier()
    dist.destroy_process_group()
    open(os.path.join(tmp, "ok%d" % rank), "w").write("ok")


def _dp_worker(rank, world, port, tmp):
    """data-parallel training (pykg2vec_b200/trainer.py): both exchange modes leave every rank with the same
    tables, equal (to fp32 rounding) to ONE process stepping on the concatenated global batch."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.dirname(here))
    sys.path.insert(0, here)
    import torch.distributed as dist
    import pykg2vec_b200
    from pykg2vec_b200 import sharding
    from pykg2vec_b200.synthetic import SyntheticConfig, SyntheticKnowledgeGraph
    from pykg2vec_b200.trainer import Trainer
    torch.cuda.set_device(rank)
    sharding.init_distributed(backend="nccl")
    dev = torch.device("cuda", rank)
    kg = SyntheticKnowledgeGraph(500, 7, 3000, 50, 50, seed=1)

    def make(model_name, opt, mode):
        cfg = SyntheticConfig(kg, device=dev, optimizer=opt, learning_rate=0.05, hidden_size=64,
                              margin=6.0 if model_name == "rotate" else 1.0, l1_flag=False, lmbda=0.01,
                              neg_rate=4 if model_name == "rotate" else 1, alpha=0.5, batch_size=128, dp_mode=mode)
        torch.manual_seed(0)
        tr = Trainer(pykg2vec_b200.import_model(model_name)(**cfg.__dict__), cfg)
        tr.build_model()
        return tr

    B = 128
    for model_name, opt in (("transe", "sgd"), ("transe", "adam"), ("distmult", "adam"), ("complex", "adagrad"), ("rotate", "adam")):
        single = make(model_name, opt, "off")
        trs = {mode: make(model_name, opt, mode) for mode in ("grads", "ids")}
        for mode, t_ in trs.items():
            t_.model.load_state_dict(single.model.state_dict())
            assert t_._dp == mode and t_._fused and single._dp is None
        for step in range(3):
            per_rank = []
            for rk in range(world):
                rng = np.random.RandomState(100 * step + rk)
                if single.model.training_strategy.name == "PAIRWISE_BASED":
                    nr = single.config.neg_rate
                    per_rank.append([rng.randint(500, size=B), rng.randint(7, size=B), rng.randint(500, size=B),
                                     rng.randint(500, size=B * nr), rng.randint(7, size=B * nr), rng.randint(500, size=B * nr)])
                else:
                    per_rank.append([rng.randint(500, size=B), rng.randint(7, size=B), rng.randint(500, size=B),
                                     np.where(np.arange(B) % 2 == 0, 1, -1)])
            to = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(dev)
            glob = [to(np.concatenate([per_rank[rk][k] for rk in range(world)])) for k in range(len(per_rank[0]))]
            # (RotatE: the negatives of positive i stay contiguous under this rank-major concatenation)
            l_single = float(single.train_batch_device(glob).item())
            for mode, t_ in trs.items():
                l_dp = float(t_.train_batch_device([to(a) for a in per_rank[rank]]).item())
                assert abs(l_dp - l_single) <= 2e-4 * max(abs(l_single), 1e-6), (model_name, opt, mode, step, l_dp, l_single)
        for mode, t_ in trs.items():
            for (ka, va), (kb, vb) in zip(t_.model.state_dict().items(), single.model.state_dict().items()):
                d1 = (va - vb).abs()
                if opt == "sgd":
                    assert float(d1.max()) <= 3e-5, (model_name, opt, mode, ka, float(d1.max()))
                else:   # (see below: a cancelling gradient element may flip a +-lr step under Adagrad / Adam)
                    assert float((d1 > 3e-5).float().mean()) <= 1e-3, (model_name, opt, mode, ka)
                # "grads": every rank applies the SAME all-reduced gradient -> replicas stay bit-identical;
                # "ids": every rank accumulates the global batch itself with float atomics (unordered): the
                # gradients agree to rounding.  SGD carries the rounding through (replicas within 1e-6); Adagrad /
                # Adam divide by a gradient magnitude, so an element whose contributions cancel can step by ~lr in
                # opposite directions — which is why Trainer._pick_dp_mode never picks "ids" for them; forced here,
                # all but a handful of elements must still agree
                other = va.clone()
                dist.broadcast(other, src=0)
                diff = (other - va).abs()
                if mode == "grads":
                    assert torch.equal(other, va), (model_name, opt, mode, ka)
                elif opt == "sgd":
                    assert float(diff.max()) <= 1e-6, (model_name, opt, mode, ka)
                else:
                    assert float((diff > 1e-6).float().mean()) <= 1e-3, (model_name, opt, mode, ka)
                    assert float(diff.max()) <= 3 * 2 * 0.05 + 1e-6, (model_name, opt, mode, ka)   # 3 steps of +-lr
        if opt != "sgd":   # left to itself the trainer keeps replicas bit-identical for these optimizers
            assert make(model_name, opt, None)._dp == "grads", (model_name, opt)
    # host API (Trainer.train_batch: pinned H2D, graph replay, D2H of the loss) in "ids" mode: the H2D copy and
    # the id all-gather are eager, the step on the gathered batch is a CUDA graph — same tables as one process
    # stepping on the concatenated batch through ITS graph
    single = make("transe", "sgd", "off")
    dp = make("transe", "sgd", "ids")
    dp.model.load_state_dict(single.model.state_dict())
    for step in range(4):
        per_rank = []
        for rk in range(world):
            rng = np.random.RandomState(7000 + 10 * step + rk)
            per_rank.append([rng.randint(500 if k % 3 != 1 else 7, size=B) for k in range(6)])
        glob = [np.concatenate([per_rank[rk][k] for rk in range(world)]) for k in range(6)]
        l_single = single.train_batch(glob)
        l_dp = float(dp.train_batch(per_rank[rank], sync=(step % 2 == 0)))
        assert abs(l_dp - l_single) <= 2e-4 * max(abs(l_single), 1e-6), (step, l_dp, l_single)
    assert any(len(k) == 2 for k in dp._graphs), "the data-parallel host step must be graph-staged"
    for (ka, va), (kb, vb) in zip(dp.model.state_dict().items(), single.model.state_dict().items()):
        assert float((va - vb).abs().max()) <= 3e-5, ka
    dist.barrier()
    dist.destroy_process_group()
    open(os.path.join(tmp, "dp_ok%d" % rank), "w").write("ok")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_data_parallel_training_nccl(tmp_path):
    world = 2
    mp.start_processes(_dp_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True,
                       start_method="spawn")
    assert all(os.path.exists(os.path.join(str(tmp_path), "dp_ok%d" % r)) for r in range(world))


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_row_sharded_and_query_sharded_eval_nccl(tmp_path):
    world = 2
    mp.start_processes(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True,
                       start_method="spawn")
    assert all(os.path.exists(os.path.join(str(tmp_path), "ok%d" % r)) for r in range(world))
