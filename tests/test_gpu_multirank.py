"""Two ranks on two GPUs over NCCL (run with `python -m pytest tests/test_gpu_multirank.py -m gpu` on a machine with
two GPUs; skipped with one): the data-parallel step on the DEVICE -- sharded queries + summed gradients == the
single-GPU full-batch step, replicas stay bit-identical, SyncBN makes batch-level BN shard-invariant, and the overlapped
all-reduce changes nothing."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _batch(B, n, F, seed):
    rng = np.random.default_rng(seed)
    p = np.array([1940952, 1225770, 504958, 69010, 30435], dtype=np.float64); p /= p.sum()
    X = rng.standard_normal((B, n, F)).astype(np.float32)
    y = rng.choice(5, size=(B, n), p=p).astype(np.float32)
    y[:, 0] = np.maximum(y[:, 0], 1.0)
    return torch.from_numpy(X), torch.from_numpy(-np.sort(-y, axis=1))


def _ranker(bn_type, dev, seed):
    import ptranking_b200
    sf = dict(sf_id="pointsf", opt="Adam", lr=1e-3,
              pointsf=dict(num_features=136, num_layers=3, AF="GE", TL_AF="S", apply_tl_af=True, BN=True, bn_type=bn_type,
                           bn_affine=True, dropout=0.0))
    torch.manual_seed(seed)
    r = ptranking_b200.LambdaRank(sf_para_dict=sf, model_para_dict=dict(model_id="LambdaRank", sigma=1.0), gpu=True, device=dev)
    return r


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _worker(rank, world, port, mode):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    os.environ["PTRANKING_B200_PEER"] = "0"       # this worker checks the NCCL path: the reduced gradient stays inspectable
    from ptranking_b200 import dist as b200dist, LABEL_TYPE
    b200dist.init_from_env("nccl")
    dev = f"cuda:{rank}"
    kw = dict(presort=True, label_type=LABEL_TYPE.MultiLabel)
    bn_type = "BN2" if mode == "bn2" else "BN"
    b200dist.set_sync_bn(mode == "syncbn")
    B, n, F = 16, 96, 136
    X, y = _batch(B, n, F, seed=5)
    shard = list(b200dist.shard_queries(B, rank, world))
    # data-parallel replica: DIFFERENT seeds per rank -- config_optimizer must broadcast rank 0's weights
    r = _ranker(bn_type, dev, seed=100 + rank)
    r.init()
    flat0 = r.grad_bucket.flat_param.clone()
    gathered = [torch.empty_like(flat0) for _ in range(world)]
    dist.all_gather(gathered, flat0)
    assert all(torch.equal(g, gathered[0]) for g in gathered), "replicas must start from identical weights"
    # the single-GPU comparator on every rank: same initial weights, the whole batch, no collectives
    full = _ranker(bn_type, dev, seed=1)
    b200dist.set_sync_bn(False)
    full.init()
    b200dist.set_sync_bn(mode == "syncbn")
    full.grad_bucket.distributed = False
    full.point_sf.load_state_dict({k: v.clone() for k, v in r.point_sf.state_dict().items()})
    r.eval_mode(); full.eval_mode()
    for step in range(2):
        l_sh, _ = r.train_op(X[shard].to(dev), y[shard].to(dev), **kw)
        # force the comparator's scorer to local statistics regardless of the global sync flag
        b200dist.set_sync_bn(False)
        l_full, _ = full.train_op(X.to(dev), y.to(dev), **kw)
        b200dist.set_sync_bn(mode == "syncbn")
        tot = l_sh.detach().clone().reshape(1)
        dist.all_reduce(tot)
        g_sh, g_full = r.grad_bucket.flat, full.grad_bucket.flat
        if mode in ("bn2", "syncbn"):
            assert abs(float(tot) - float(l_full)) <= 2e-5 * abs(float(l_full)), (mode, step, float(tot), float(l_full))
            assert _rel(g_sh, g_full) <= 5e-5, (mode, step, _rel(g_sh, g_full))
        else:       # plain BN under sharding normalises with per-rank statistics: a different computation
            assert _rel(g_sh, g_full) > 1e-3
        # replicas stay bit-identical step after step
        dist.all_gather(gathered, r.grad_bucket.flat_param)
        assert all(torch.equal(g, gathered[0]) for g in gathered), (mode, step)
    if mode in ("bn2", "syncbn"):
        assert _rel(r.grad_bucket.flat_param, full.grad_bucket.flat_param) <= 2e-3
    # overlapped all-reduce == single all-reduce (bit for bit with two ranks)
    os.environ["PTRANKING_B200_OVERLAP"] = "0"
    a = _ranker(bn_type, dev, seed=7); a.init(); a.eval_mode()
    os.environ["PTRANKING_B200_OVERLAP"] = "1"
    b = _ranker(bn_type, dev, seed=7); b.init(); b.eval_mode()
    os.environ["PTRANKING_B200_OVERLAP"] = "0"
    a.train_op(X[shard].to(dev), y[shard].to(dev), **kw)
    os.environ["PTRANKING_B200_OVERLAP"] = "1"
    b.train_op(X[shard].to(dev), y[shard].to(dev), **kw)
    assert b.grad_bucket._side is not None, "the overlapped path did not engage"
    assert torch.equal(a.grad_bucket.flat, b.grad_bucket.flat)
    torch.cuda.synchronize()
    dist.destroy_process_group()


def _peer_worker(rank, world, port, opt):
    """The gradient sum inside the optimizer kernel (NVLink peer memory, csrc/optim.cu) against the NCCL all-reduce +
    step it replaces: same weights after every step (two ranks: a + b is order-free, so bit for bit), replicas identical,
    the bare exchange equals dist.all_reduce, and no rank ever timed out."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import ptranking_b200
    from ptranking_b200 import dist as b200dist, ops, LABEL_TYPE
    b200dist.init_from_env("nccl")
    dev = f"cuda:{rank}"
    kw = dict(presort=True, label_type=LABEL_TYPE.MultiLabel)
    B, n, F = 16, 96, 136
    X, y = _batch(B, n, F, seed=9)
    shard = list(b200dist.shard_queries(B, rank, world))
    Xs, ys = X[shard].to(dev), y[shard].to(dev)

    def make(peer):
        os.environ["PTRANKING_B200_PEER"] = "1" if peer else "0"
        sf = dict(sf_id="pointsf", opt=opt, lr=1e-3,
                  pointsf=dict(num_features=136, num_layers=3, AF="GE", TL_AF="S", apply_tl_af=True, BN=True, bn_type="BN2",
                               bn_affine=True, dropout=0.0))
        torch.manual_seed(3)
        r = ptranking_b200.LambdaRank(sf_para_dict=sf, model_para_dict=dict(model_id="LambdaRank", sigma=1.0), gpu=True, device=dev)
        r.init(); r.eval_mode()
        return r

    a, b = make(True), make(False)
    assert a.grad_bucket.peer is not None, "the peer exchange did not engage"
    assert b.grad_bucket.peer is None
    gathered = [torch.empty_like(a.grad_bucket.flat_param) for _ in range(world)]
    for step in range(4):
        la, _ = a.train_op(Xs, ys, **kw)
        lb, _ = b.train_op(Xs, ys, **kw)
        assert torch.equal(la, lb), (opt, step)
        assert torch.equal(a.grad_bucket.flat_param, b.grad_bucket.flat_param), (opt, step)
        dist.all_gather(gathered, a.grad_bucket.flat_param)
        assert all(torch.equal(g, gathered[0]) for g in gathered), (opt, step)
    # the bare exchange on the same mapped buffers
    ex = a.grad_bucket.peer
    k = a.grad_bucket._peer_k
    torch.manual_seed(50 + rank)
    ex.bufs[k].copy_(torch.randn(ex.count, device=dev))
    ref = ex.bufs[k].clone()
    dist.all_reduce(ref)
    torch.cuda.synchronize(); dist.barrier()
    out = ops.peer_allreduce_sum(torch.empty_like(ref), ex.group(k))
    assert torch.equal(out, ref)
    assert ex.error() == 0
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("opt", ["Adam", "Adagrad", "RMS"])
def test_two_rank_peer_memory_step_equals_nccl_step(opt):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    mp.spawn(_peer_worker, args=(2, _free_port(), opt), nprocs=2, join=True)


@pytest.mark.parametrize("mode", ["bn2", "syncbn", "bn_local"])
def test_two_rank_step_equals_full_batch(mode):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    mp.spawn(_worker, args=(2, _free_port(), mode), nprocs=2, join=True)
