"""The device DIVDataset: its orders, rows and matrices against the unmodified reference (tests/golden/divdata.npz) and
the float64 greedy restatement, one launch for a whole split against one launch per query, n = 4096, the noise stream,
and one training epoch plus evaluation on a device split against the same ranker on the reference's split."""
import copy

import numpy as np
import pytest
import torch

from tests import daletor_oracle as do
from tests import divdata_oracle as oracle
from tests.helpers import load

DEV = "cuda:0"
gpu = pytest.mark.gpu


def _dataset(dicts, qids=None, **kw):
    from ptranking_b200.ltr_diversification.div_data import DIVDataset
    all_qids, q_reprs, doc_reprs, perms, q_docs = dicts
    return DIVDataset(split_type=None, list_as_file=all_qids if qids is None else qids,
                      data_dict=dict(data_id="WT_Div_0912_Implicit"), fold_dir="unused/", presort=True,
                      dictQueryRepresentation=q_reprs, dictDocumentRepresentation=doc_reprs, dictQueryPermutaion=perms,
                      dictQueryDocumentSubtopics=q_docs, device=DEV, **kw)


def _random_dicts(rng, lens, F=8, p_absent=0.1, p_empty=0.05):
    """TREC-shaped dicts: query q's pool of lens[q] documents drawn from one shared table, string subtopic ids 1..20."""
    D = max(lens) + 500
    doc_reprs = {f"d{r}": rng.standard_normal((1, F)) for r in range(D)}
    q_reprs, perms, q_docs = {}, {}, {}
    for q, n in enumerate(lens):
        pool = [f"d{r}" for r in rng.choice(D, size=n, replace=False)]
        ids = np.sort(rng.choice(np.arange(1, 21), size=int(rng.integers(1, 21)), replace=False))
        subs = {}
        for doc in pool:
            u = rng.random()
            if u < p_absent:
                continue
            subs[doc] = [] if u < p_absent + p_empty else [str(s) for s in ids if rng.random() < 0.3]
        q_reprs[str(q)], perms[str(q)], q_docs[str(q)] = rng.standard_normal((1, F)), \
            dict(alphaDCG=0.0, permutation=pool), subs
    return list(range(len(lens))), q_reprs, doc_reprs, perms, q_docs


def _check_against_oracle(ds, dicts):
    """Every query: the device order is the oracle's (lowest position on ties), each pick has the largest remaining
    gain, and the rows, matrix and perm_docs are the pool gathered in that order."""
    qids, q_reprs, doc_reprs, perms, q_docs = dicts
    orders = []
    for b, qid in enumerate(ds._host.qids):
        pool, cover = oracle.pool_covers(perms, q_docs, qid)
        t, q, perm_docs, docs, alpha_dcg, subtopics, R = ds[b]
        o0, o1 = ds._host.offsets[b], ds._host.offsets[b + 1]
        order = ds.order[o0:o1]
        want, picked, best, _ = oracle.replay(cover, order=order)
        np.testing.assert_array_equal(picked, best, err_msg=f"query {qid}")
        np.testing.assert_array_equal(order, oracle.replay(cover)[0], err_msg=f"query {qid}")
        assert t == qid and perm_docs == [pool[i] for i in order] and subtopics is q_docs[str(qid)]
        assert alpha_dcg == perms[str(qid)]["alphaDCG"]
        rows = np.vstack([doc_reprs[d] for d in perm_docs]).astype(np.float32)
        assert np.array_equal(docs.cpu().numpy(), rows)
        assert np.array_equal(q.cpu().numpy(), np.asarray(q_reprs[str(qid)], dtype=np.float32).reshape(1, -1))
        assert np.array_equal(R.cpu().numpy(), oracle.to_matrix(cover, order))
        orders.append(order)
    return orders


@gpu
def test_fixture_parity():
    z = load("divdata.npz")
    dicts = oracle.input_dicts(z)
    ds = _dataset(dicts)
    orders = _check_against_oracle(ds, dicts)
    exact = 0
    for b, qid in enumerate(dicts[0]):
        ref, order = z[f"ref_order_{qid}"], orders[b]
        _, docs_t, _, docs, _, _, R = ds[b]
        pool, cover = oracle.pool_covers(dicts[3], dicts[4], qid)
        if oracle.tie_free(cover, ref):
            np.testing.assert_array_equal(order, ref, err_msg=f"tie-free query {qid}")
            exact += 1
        # the reference's rows and columns, gathered in the device order
        where = np.argsort(ref)[order]
        assert np.array_equal(docs.cpu().numpy(), z[f"ref_docs_{qid}"][where])
        assert np.array_equal(R.cpu().numpy(), z[f"ref_rele_{qid}"][:, where])
        assert np.array_equal(docs_t.cpu().numpy(), z[f"q_{qid}"].astype(np.float32))
    assert exact >= 12


@gpu
def test_one_launch_for_200_queries_is_bitwise_the_one_query_launches():
    rng = np.random.default_rng(7)
    dicts = _random_dicts(rng, [int(n) for n in rng.integers(1, 400, 200)])
    whole = _dataset(dicts)
    _check_against_oracle(whole, dicts)
    for b, qid in enumerate(dicts[0]):
        one = _dataset(dicts, [qid])
        assert np.array_equal(one.order, whole.order[whole._host.offsets[b]:whole._host.offsets[b + 1]])
        for x, y in zip(one[0], whole[b]):
            if isinstance(x, torch.Tensor):
                assert torch.equal(x, y), qid
            else:
                assert x == y or x is y


@gpu
def test_4096_documents_20_subtopics():
    rng = np.random.default_rng(8)
    dicts = _random_dicts(rng, [4096, 4096, 17], p_absent=0.02, p_empty=0.01)
    for q in ("0", "1"):
        subs = dicts[4][q]
        for doc in list(subs)[:20]:
            subs[doc] = [str(s) for s in range(1, 21)]          # every id present
    ds = _dataset(dicts)
    _check_against_oracle(ds, dicts)
    assert ds[0][6].shape == (20, 4096) and ds[1][6].shape == (20, 4096)


@gpu
def test_noise_is_deterministic_per_seed_and_standard_normal():
    rng = np.random.default_rng(9)
    dicts = _random_dicts(rng, [int(n) for n in rng.integers(50, 400, 60)], F=16)
    clean = _dataset(dicts)
    a = _dataset(dicts, add_noise=True, std_delta=0.5, noise_seed=1234)
    b = _dataset(dicts, add_noise=True, std_delta=0.5, noise_seed=1234)
    c = _dataset(dicts, add_noise=True, std_delta=0.5, noise_seed=1235)
    assert torch.equal(a.q, b.q) and torch.equal(a.docs, b.docs)
    assert not torch.equal(a.docs, c.docs) and not torch.equal(a.q, c.q)
    numel = clean._host.rele_numel
    assert torch.equal(a.rele.rele[:numel], clean.rele.rele[:numel]) and np.array_equal(a.order, clean.order)
    torch.manual_seed(5)
    d = _dataset(dicts, add_noise=True, std_delta=0.5)
    torch.manual_seed(5)
    e = _dataset(dicts, add_noise=True, std_delta=0.5)
    assert d.noise_seed == e.noise_seed and torch.equal(d.docs, e.docs)
    noise = torch.cat([(a.docs - clean.docs).reshape(-1), (a.q - clean.q).reshape(-1)]).double() / 0.5
    N = noise.numel()
    assert N > 100000
    assert abs(float(noise.mean())) < 5.0 / N ** 0.5
    assert abs(float(noise.std()) - 1.0) < 5.0 * (2.0 / N) ** 0.5
    assert abs(float((noise.abs() < 1.0).double().mean()) - 0.682689) < 0.005


def _ranker(model_id, sf_id, F):
    import ptranking_b200
    from tests import divlist_oracle as dl
    if sf_id == "pointsf":
        sf = dict(sf_id="pointsf", opt="Adagrad", lr=0.01,
                  pointsf=dict(num_features=F, h_dim=16, num_layers=2, AF="R", TL_AF="S", apply_tl_af=False, BN=True,
                               bn_type="BN", bn_affine=True, dropout=0.1))
    else:
        sf = dict(sf_id="listsf", opt="Adagrad", lr=0.01,
                  listsf=dict(num_features=F, **dict(dl.SMALL_LISTSF, encoder_type="AttnDIN", n_heads=2)))
    mp = dict(model_id="DALETOR", rt=10.0, top_k=10) if model_id == "DALETOR" else \
        dict(model_id="DivProbRanker", K=1, cluster=False, sort_id="ExpRele", limit_delta=0.01, opt_id="SuperSoft",
             metric="nERR-IA", top_k=None, opt_ideal=True, norm=True)
    torch.manual_seed(77)
    r = ptranking_b200.DIV_MODELS[model_id](sf_para_dict=copy.deepcopy(sf), model_para_dict=mp, gpu=True, device=DEV)
    r.init()
    if sf_id == "pointsf":
        init = do.seeded_state({k: tuple(v.shape) for k, v in r.point_sf.state_dict().items()})
        with torch.no_grad():
            for k, v in r.point_sf.state_dict().items():
                v.copy_(torch.from_numpy(init[k]))
    return r


def _state(r):
    if r.sf_id == "pointsf":
        return r.point_sf.state_dict()
    return {f"{p}.{k}": v for p, part in r.list_sf.items() for k, v in part.state_dict().items()}


@gpu
@pytest.mark.parametrize("sf_id", ["pointsf", "listsf"])
@pytest.mark.parametrize("model_id", ["DALETOR", "DivProbRanker"])
def test_epoch_on_a_device_split_is_the_epoch_on_the_reference_split(model_id, sf_id):
    """The queries whose reference order has no tie, built on the device and, as the reference built them, fed from
    the host: one epoch with dropout and one evaluation give the same losses, parameters and metrics, bit for bit."""
    from ptranking_b200 import ops
    z = load("divdata.npz")
    dicts = oracle.input_dicts(z)
    qids = [q for q in dicts[0] if oracle.tie_free(oracle.pool_covers(dicts[3], dicts[4], q)[1], z[f"ref_order_{q}"])]
    assert len(qids) >= 12
    ds = _dataset(dicts, qids)
    host = [(q, torch.from_numpy(z[f"q_{q}"]).float(), None, torch.from_numpy(z[f"ref_docs_{q}"]), 0.0, None,
             torch.from_numpy(z[f"ref_rele_{q}"])) for q in qids]
    F = z["table"].shape[1]
    a, b = _ranker(model_id, sf_id, F), _ranker(model_id, sf_id, F)
    for (ka, pa), (kb, pb) in zip(_state(a).items(), _state(b).items()):
        assert ka == kb and torch.equal(pa, pb), ka
    o0 = ops._dropout_offset
    loss_a, stop_a = a.div_train(ds, epoch_k=1)
    ops._dropout_offset = o0
    loss_b, stop_b = b.div_train(host, epoch_k=1)
    assert stop_a == stop_b
    assert torch.equal(loss_a, loss_b), (float(loss_a), float(loss_b))
    for (ka, pa), (kb, pb) in zip(_state(a).items(), _state(b).items()):
        assert torch.equal(pa, pb), ka
    res_a = a.srd_performance_at_ks(test_data=ds, ks=[1, 3, 5], max_label=1.0)
    res_b = b.srd_performance_at_ks(test_data=host, ks=[1, 3, 5], max_label=1.0)
    for x, y in zip(res_a, res_b):
        assert torch.equal(x, y)
    assert torch.equal(a.alpha_ndcg_at_k(test_data=ds, k=3), b.alpha_ndcg_at_k(test_data=host, k=3))


@gpu
def test_bad_arguments_are_refused_before_launch():
    from ptranking_b200 import _lib
    lib = _lib.load()
    buf = torch.zeros(64, dtype=torch.int32, device=DEV)
    p = buf.data_ptr()
    n0 = lib.ptrb200_launch_count()
    assert lib.ptrb200_div_ideal_order(None, p, p, p, 2, 5, p, None) != 0
    assert lib.ptrb200_div_ideal_order(p, p, p, p, 0, 5, p, None) != 0
    assert lib.ptrb200_div_ideal_order(p, p, p, p, 2, 4097, p, None) != 0
    assert b"PTRB200_MAX_LIST_LEN" in lib.ptrb200_last_error()
    args = [p, 4, p, p, p, p, p, p, p, p, 2, 0.0, 0, p, p, p, None]
    for i, bad in ((0, None), (1, 0), (10, 0), (11, -1.0), (11, float("inf")), (14, None)):
        call = list(args)
        call[i] = bad
        assert lib.ptrb200_div_pack_split(*call) != 0, i
    assert lib.ptrb200_launch_count() == n0
