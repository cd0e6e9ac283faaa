"""CPU checks of the device DIVDataset: the float64 greedy restatement against the unmodified reference's splits
(tests/golden/divdata.npz), the host index and subtopic CSR the kernels read, the refusals (raised before any device
work) and the opt-in installer."""
import types

import numpy as np
import pytest

from tests import divdata_oracle as oracle
from tests.helpers import load


@pytest.fixture(scope="module")
def z():
    return load("divdata.npz")


@pytest.fixture(scope="module")
def dicts(z):
    return oracle.input_dicts(z)


def test_fixture_shapes(z, dicts):
    qids, _, _, perms, q_docs = dicts
    lens = [len(oracle.pool_covers(perms, q_docs, q)[0]) for q in qids]
    assert min(lens) == 1 and max(lens) == 4000 and sum(300 <= n <= 450 for n in lens) >= 2
    covers = [c for q in qids for c in oracle.pool_covers(perms, q_docs, q)[1]]
    assert any(c is None for c in covers) and any(c == [] for c in covers)
    assert max(s for c in covers if c for s in c) == 20


def test_reference_orders_are_greedy_and_match_the_oracle_where_tie_free(z, dicts):
    """Every reference pick has the largest remaining gain; where its order meets no tie the oracle's order is it."""
    qids, _, _, perms, q_docs = dicts
    tie_free = 0
    for q in qids:
        _, cover = oracle.pool_covers(perms, q_docs, q)
        ref = z[f"ref_order_{q}"]
        assert sorted(ref.tolist()) == list(range(len(cover)))
        _, picked, best, ties = oracle.replay(cover, order=ref)
        np.testing.assert_array_equal(picked, best, err_msg=f"query {q}")
        if np.all(ties == 1):
            tie_free += 1
            np.testing.assert_array_equal(oracle.replay(cover)[0], ref, err_msg=f"query {q}")
    assert tie_free >= 12


def test_reference_rows_and_matrices_are_the_pool_in_its_order(z, dicts):
    qids, _, _, perms, q_docs = dicts
    table = z["table"]
    for q in qids:
        pool, cover = oracle.pool_covers(perms, q_docs, q)
        ref = z[f"ref_order_{q}"]
        rows = np.asarray([int(d[1:]) for d in pool])[ref]
        np.testing.assert_array_equal(z[f"ref_docs_{q}"], table[rows].astype(np.float32))
        np.testing.assert_array_equal(z[f"ref_rele_{q}"], oracle.to_matrix(cover, ref))
    # a pool without any subtopic gives 19 zero rows
    empty = [q for q in qids if all(not c for c in oracle.pool_covers(perms, q_docs, q)[1])]
    assert empty and all(z[f"ref_rele_{q}"].shape[0] == 19 and not z[f"ref_rele_{q}"].any() for q in empty)


def test_host_split_index_and_csr(z, dicts):
    from ptranking_b200.ltr_diversification.div_data import HostSplit, doc_table
    qids, q_reprs, doc_reprs, perms, q_docs = dicts
    table = doc_table(doc_reprs)
    h = HostSplit(qids, table, q_reprs, perms, q_docs)
    assert len(h) == len(qids)
    np.testing.assert_array_equal(table.rows(), z["table"].astype(np.float32))
    for b, q in enumerate(qids):
        pool, cover = oracle.pool_covers(perms, q_docs, q)
        o0, o1 = h.offsets[b], h.offsets[b + 1]
        assert h.pools[b] == pool and o1 - o0 == len(pool)
        np.testing.assert_array_equal(h.rows[o0:o1], [int(d[1:]) for d in pool])
        for i, c in enumerate(cover):
            e0, e1 = h.sub_offsets[o0 + i], h.sub_offsets[o0 + i + 1]
            assert h.sub_ids[e0:e1].tolist() == (c or [])
        R = oracle.to_matrix(cover, np.arange(len(pool)))
        assert h.sub_counts[b] == R.shape[0] and h.rele_sum[b] == R.sum()
        assert h.rele_offsets[b] == sum(int(h.sub_counts[k]) * len(h.pools[k]) for k in range(b))
        np.testing.assert_array_equal(h.q_rows[b], z[f"q_{q}"][0].astype(np.float32))
        assert h.alpha_dcgs[b] == float(q) and h.subtopics[b] is q_docs[str(q)]
    assert h.max_nnz == max(int(h.sub_offsets[h.offsets[b + 1]] - h.sub_offsets[h.offsets[b]]) for b in range(len(h)))
    assert h.rele_numel == sum(int(h.sub_counts[b]) * len(h.pools[b]) for b in range(len(h)))


def test_doc_table_is_shared_per_dict_object(dicts):
    from ptranking_b200.ltr_diversification.div_data import doc_table
    doc_reprs = dicts[2]
    t = doc_table(doc_reprs)
    assert doc_table(doc_reprs) is t
    other = dict(doc_reprs)
    assert doc_table(other) is not t


def test_alpha_powers_are_the_reference_terms():
    from ptranking_b200.ltr_diversification.div_data import alpha_powers
    for alpha in (0.5, 0.3, 0.9):
        pw = alpha_powers(alpha, 300)
        assert pw.dtype == np.float64 and pw.size == 300
        for c in (0, 1, 7, 299):
            assert pw[c] == (1 - alpha) ** np.float64(c)


def _kw(dicts, **over):
    qids, q_reprs, doc_reprs, perms, q_docs = dicts
    kw = dict(split_type=None, list_as_file=qids[:5], data_dict=dict(data_id="WT_Div_0912_Implicit"), fold_dir="x/",
              presort=True, dictQueryRepresentation=q_reprs, dictDocumentRepresentation=doc_reprs,
              dictQueryPermutaion=perms, dictQueryDocumentSubtopics=q_docs, buffer=True)
    kw.update(over)
    return kw


@pytest.fixture
def no_device(monkeypatch):
    """Any device work (loading the library, uploading the table, asking for the CUDA device) fails the test."""
    from ptranking_b200 import _lib
    from ptranking_b200.ltr_diversification import div_data

    def boom(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(_lib, "load", boom)
    monkeypatch.setattr(div_data._DocTable, "on", boom)
    monkeypatch.setattr(div_data.torch.cuda, "current_device", boom)


def test_refusals_come_before_device_work(dicts, no_device):
    import copy
    from ptranking_b200.ltr_diversification.div_data import DIVDataset
    qids, q_reprs, doc_reprs, perms, q_docs = dicts
    with pytest.raises(AssertionError, match="presort"):
        DIVDataset(**_kw(dicts, presort=False))
    with pytest.raises(NotImplementedError):
        DIVDataset(**_kw(dicts, data_dict=dict(data_id="MQ2007")))
    bad_perm = copy.deepcopy(perms)
    bad_perm["2"]["permutation"] = bad_perm["2"]["permutation"] + ["no-such-doc"]
    with pytest.raises(ValueError, match="no-such-doc"):
        DIVDataset(**_kw(dicts, dictQueryPermutaion=bad_perm))
    bad_perm["2"]["permutation"] = []
    with pytest.raises(ValueError, match="empty permutation"):
        DIVDataset(**_kw(dicts, dictQueryPermutaion=bad_perm))
    for sid in ("0", "21", "-3"):
        bad = copy.deepcopy(q_docs)
        doc = perms["4"]["permutation"][0]
        bad["4"][doc] = ["1", sid]
        with pytest.raises(ValueError, match=f"subtopic id {int(sid)} outside 1..20"):
            DIVDataset(**_kw(dicts, dictQueryDocumentSubtopics=bad))
    with pytest.raises(ValueError, match="std_delta"):
        DIVDataset(**_kw(dicts, add_noise=True, std_delta=-1.0))
    with pytest.raises(ValueError, match="PTRB200_MAX_LIST_LEN"):
        long = copy.deepcopy(perms)
        long["0"]["permutation"] = list(doc_reprs)[:4097]
        DIVDataset(**_kw(dicts, dictQueryPermutaion=long))


def test_install_div_data_sets_only_the_dataset_class():
    import ptranking_b200
    from ptranking_b200.ltr_diversification.div_data import DIVDataset
    old = object()
    module = types.SimpleNamespace(DIVDataset=old, RerankDIVDataset="rerank", DALETOR="d", DivProbRanker="p")
    before = dict(vars(module))
    assert ptranking_b200.install_div_data(module) == {"DIVDataset": old}
    assert module.DIVDataset is DIVDataset
    assert {k: v for k, v in vars(module).items() if k != "DIVDataset"} == \
        {k: v for k, v in before.items() if k != "DIVDataset"}
    module2 = types.SimpleNamespace(DIVDataset=old)
    ptranking_b200.install_diversification(module2)
    assert module2.DIVDataset is old
