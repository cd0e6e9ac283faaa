"""Rerank mode on the device: the select and gather kernels against NumPy, the CUDA first stages against the
unmodified reference's RerankDIVDataset (tests/golden/div_rerank.npz), second-stage epochs on a device selection against
the same epochs fed the reference's pools from the host, fresh selections under dropout, and argument refusal."""
import copy

import numpy as np
import pytest
import torch

from tests import daletor_oracle as do
from tests.helpers import load
from tests.rerank_oracle import F, KS, STAGES, pool_queries, stage_config, topk_ascending

DEV = "cuda:0"
gpu = pytest.mark.gpu


def _offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def _select(keys_list, k, total=True):
    from ptranking_b200 import ops
    lens = [len(x) for x in keys_list]
    keys = torch.from_numpy(np.concatenate(keys_list).astype(np.float32)).to(DEV)
    offs = torch.from_numpy(_offsets(lens)).to(DEV)
    tot = int(np.minimum(lens, k).sum()) if total else None
    counts, so, idx = ops.div_rerank_select(keys, offs, max(lens), k, total=tot)
    return counts.cpu().numpy(), so.cpu().numpy(), idx.cpu().numpy()


def _key_cases(rng):
    yield "random", [rng.standard_normal(int(n)).astype(np.float32) for n in rng.integers(1, 301, 40)], (1, 5, 50, 400)
    ties = [rng.integers(0, 3, int(n)).astype(np.float32) for n in rng.integers(1, 200, 30)]
    ties.append(np.asarray([0.0, -0.0, 0.0, -0.0, 1.0], dtype=np.float32))
    yield "ties", ties, (1, 2, 3, 7, 64)
    yield "all_equal", [np.full(int(n), 0.5, dtype=np.float32) for n in (1, 7, 100, 513)], (1, 5, 100, 600)
    yield "n_vs_k", [rng.standard_normal(n).astype(np.float32) for n in (3, 5, 5, 10, 4, 6)], (5,)
    yield "long_ragged", [np.round(rng.standard_normal(n), 1).astype(np.float32)
                          for n in (4096, 1, 4095, 2048, 3000, 17, 4096)], (1, 100, 4000, 4096)


@gpu
def test_select_matches_numpy_total_order():
    rng = np.random.default_rng(11)
    for name, keys_list, ks in _key_cases(rng):
        for k in ks:
            counts, so, idx = _select(keys_list, k)
            assert so[0] == 0 and so[-1] == idx.size
            for q, keys in enumerate(keys_list):
                want = topk_ascending(keys, k)
                assert counts[q] == want.size
                np.testing.assert_array_equal(idx[so[q]:so[q + 1]], want, err_msg=f"{name} k={k} query {q}")
        # the read-back total gives the same selection
        c2, so2, idx2 = _select(keys_list, ks[0], total=False)
        c1, so1, idx1 = _select(keys_list, ks[0])
        assert np.array_equal(c1, c2) and np.array_equal(so1, so2) and np.array_equal(idx1, idx2)


@gpu
def test_gather_is_bit_exact():
    from ptranking_b200 import ops
    rng = np.random.default_rng(12)
    lens = [int(n) for n in rng.integers(1, 400, 25)] + [4096]
    mats = [rng.uniform(0, 2, (int(rng.integers(1, 9)), n)).astype(np.float32) for n in lens]
    docs = rng.standard_normal((sum(lens), 7)).astype(np.float32)
    keys = [rng.standard_normal(n).astype(np.float32) for n in lens]
    for k in (1, 13, 300):
        counts, so, idx = _select(keys, k)
        rele = ops.SubtopicRele.pack([torch.from_numpy(m) for m in mats], DEV)
        d_out, r_out = ops.div_rerank_gather(torch.from_numpy(docs).to(DEV), torch.from_numpy(_offsets(lens)).to(DEV),
                                             torch.from_numpy(so).to(DEV), torch.from_numpy(idx).to(DEV), rele)
        d_out, flat = d_out.cpu().numpy(), r_out.rele.cpu().numpy()
        ro = r_out.rele_offsets.cpu().numpy()
        off = _offsets(lens)
        for q, n in enumerate(lens):
            sel = idx[so[q]:so[q + 1]]
            assert np.array_equal(d_out[so[q]:so[q + 1]], docs[off[q] + sel])
            m, c = mats[q].shape[0], sel.size
            assert np.array_equal(flat[ro[q]:ro[q] + m * c].reshape(m, c), mats[q][:, sel])


def _discriminator(stage, z):
    import ptranking_b200
    mp, sf, mode = stage_config(stage)
    r = ptranking_b200.DIV_MODELS[mp["model_id"]](sf_para_dict=sf, model_para_dict=mp, gpu=True, device=DEV)
    r.init()
    with torch.no_grad():
        for k, v in r.point_sf.state_dict().items():
            v.copy_(torch.from_numpy(z[f"{stage}__state__{k}"]))
    r.train_mode() if mode == "train" else r.eval_mode()
    return r


def _reference_pools(z, stage, k):
    """The reference's reranked lists as host tuples, with the one-document squeeze undone ([1, F] and [m, 1])."""
    out = []
    for i in range(int(z["num_queries"])):
        q, docs, R = z[f"pool_{i}__q"], z[f"pool_{i}__docs"], z[f"pool_{i}__rele"]
        if f"{stage}_k{k}_{i}__docs" in z.files:
            docs, R = z[f"{stage}_k{k}_{i}__docs"], z[f"{stage}_k{k}_{i}__rele"]
        c = docs.size // F
        out.append((f"q{i}", torch.from_numpy(q), None, torch.from_numpy(docs.reshape(c, F)), 0.0, None,
                    torch.from_numpy(R.reshape(-1, c))))
    return out


@gpu
@pytest.mark.parametrize("stage", sorted(STAGES))
def test_first_stage_reproduces_the_reference_pools(stage):
    from ptranking_b200.ltr_diversification.div_data import RerankDIVDataset
    z = load("div_rerank.npz")
    d = _discriminator(stage, z)
    pool = pool_queries(z)
    for k in KS:
        ds = RerankDIVDataset.from_queries(pool, d, k)
        sel = ds.select()
        keys = sel.keys.cpu().numpy()
        want = _reference_pools(z, stage, k)
        for i in range(len(ds)):
            o0, o1 = ds.pool().offsets_host[i:i + 2]
            assert np.abs(keys[o0:o1] - z[f"{stage}__keys_{i}"]).max() <= 1e-4 * (1 + np.abs(keys[o0:o1]).max())
            qid, _, perm_docs, docs, _, subtopics, R = ds[i]
            assert qid == f"q{i}" and perm_docs is None and subtopics is None
            assert torch.equal(docs.cpu(), want[i][3]), (k, i)
            assert torch.equal(R.cpu(), want[i][6]), (k, i)


def _second_stage(model_id):
    import ptranking_b200
    sf = dict(sf_id="pointsf", opt="Adagrad", lr=0.01,
              pointsf=dict(num_features=F, h_dim=16, num_layers=2, AF="R", TL_AF="S", apply_tl_af=False, BN=True,
                           bn_type="BN", bn_affine=True, dropout=0.1))
    mp = dict(model_id="DALETOR", rt=10.0, top_k=10) if model_id == "DALETOR" else \
        dict(model_id="DivProbRanker", K=1, cluster=False, sort_id="ExpRele", limit_delta=0.01, opt_id="SuperSoft",
             metric="nERR-IA", top_k=None, opt_ideal=True, norm=True)
    r = ptranking_b200.DIV_MODELS[model_id](sf_para_dict=copy.deepcopy(sf), model_para_dict=mp, gpu=True, device=DEV)
    r.init()
    init = do.seeded_state({k: tuple(v.shape) for k, v in r.point_sf.state_dict().items()})
    with torch.no_grad():
        for k, v in r.point_sf.state_dict().items():
            v.copy_(torch.from_numpy(init[k]))
    return r


@gpu
@pytest.mark.parametrize("qps", [1, 4])
@pytest.mark.parametrize("model_id", ["DivProbRanker", "DALETOR"])
def test_epoch_on_the_device_selection_is_the_host_fed_epoch(model_id, qps):
    """Second stage with dropout: the discriminator's forward draws one dropout offset per pass, so the host-fed arm
    starts its epoch at the offset the device arm's training started at."""
    from ptranking_b200 import ops
    from ptranking_b200.ltr_diversification.div_data import RerankDIVDataset
    z = load("div_rerank.npz")
    d = _discriminator("divprob", z)
    ds = RerankDIVDataset.from_queries(pool_queries(z), d, 50)
    host = _reference_pools(z, "divprob", 50)
    o = ops._dropout_offset
    ds.select()
    per_pass = ops._dropout_offset - o
    a, b = _second_stage(model_id), _second_stage(model_id)
    o0 = ops._dropout_offset
    loss_a, stop_a = a.div_train(ds, epoch_k=1, queries_per_step=qps)
    ops._dropout_offset = o0 + per_pass
    loss_b, stop_b = b.div_train(host, epoch_k=1, queries_per_step=qps)
    assert stop_a == stop_b
    assert torch.equal(loss_a, loss_b), (float(loss_a), float(loss_b))
    for (ka, pa), (kb, pb) in zip(a.point_sf.state_dict().items(), b.point_sf.state_dict().items()):
        assert ka == kb and torch.equal(pa, pb), ka
    res_a = a.srd_performance_at_ks(test_data=ds, ks=[1, 5, 10], max_label=1.0)
    res_b = b.srd_performance_at_ks(test_data=host, ks=[1, 5, 10], max_label=1.0)
    for x, y in zip(res_a, res_b):
        assert torch.equal(x, y)


@gpu
def test_dropout_passes_select_fresh_pools():
    """A discriminator left in training mode with dropout draws new keys on every pass; each selection is the top-k of
    its own pass's keys, recomputed through the scorer forward at that pass's dropout offset."""
    import ptranking_b200
    from ptranking_b200 import ops
    from ptranking_b200.ltr_diversification.div_data import RerankDIVDataset
    z = load("div_rerank.npz")
    mp, sf, _ = stage_config("divprob")
    sf["pointsf"]["dropout"] = 0.5
    d = ptranking_b200.DivProbRanker(sf_para_dict=sf, model_para_dict=mp, gpu=True, device=DEV)
    d.init()
    d.train_mode()
    ds = RerankDIVDataset.from_queries(pool_queries(z), d, 5)
    picks = []
    for _ in range(2):
        o = ops._dropout_offset
        sel = ds.select()
        after = ops._dropout_offset
        ops._dropout_offset = o
        keys = d.split_keys(ds.pool())
        assert ops._dropout_offset == after
        assert torch.equal(keys, sel.keys)
        keys, idx, so = keys.cpu().numpy(), sel.sel_idx.cpu().numpy(), sel.sel_offsets.cpu().numpy()
        off = ds.pool().offsets_host
        for q in range(len(ds)):
            np.testing.assert_array_equal(idx[so[q]:so[q + 1]], topk_ascending(keys[off[q]:off[q + 1]], 5))
        picks.append(idx)
    assert not np.array_equal(picks[0], picks[1])
    # a training pass over the dataset selects anew as well
    second = _second_stage("DALETOR")
    sp1, sp2 = second._split(ds), second._split(ds)
    assert sp1 is not sp2 and not torch.equal(sp1.X, sp2.X)


@gpu
def test_bad_arguments_are_refused_before_launch():
    from ptranking_b200 import _lib, ops
    keys = torch.zeros(8, device=DEV)
    offs = torch.tensor([0, 3, 8], dtype=torch.int32, device=DEV)
    lib = _lib.load()
    n0 = lib.ptrb200_launch_count()
    with pytest.raises(_lib.B200LibraryError, match="rerank_k"):
        ops.div_rerank_select(keys, offs, 5, 0)
    with pytest.raises(_lib.B200LibraryError, match="PTRB200_MAX_LIST_LEN"):
        ops.div_rerank_select(keys, offs, 4097, 3)
    p = keys.data_ptr()
    assert lib.ptrb200_div_rerank_select(None, offs.data_ptr(), 2, 5, 3, p, p, p, None, None) != 0
    assert lib.ptrb200_div_rerank_select(p, offs.data_ptr(), 2, 5, 3, p, None, p, None, None) != 0
    assert lib.ptrb200_div_rerank_select(p, offs.data_ptr(), 0, 5, 3, p, p, p, None, None) != 0
    assert lib.ptrb200_div_rerank_gather(p, 4, offs.data_ptr(), None, p, 2, p, p, p, p, p, p, None) != 0
    assert lib.ptrb200_div_rerank_gather(p, 0, offs.data_ptr(), p, p, 2, p, p, p, p, p, p, None) != 0
    assert lib.ptrb200_launch_count() == n0
