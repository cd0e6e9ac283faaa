"""CPU checks of rerank mode: the reference fixture (tests/golden/div_rerank.npz) against the NumPy restatement of the
selection, and the opt-in installer."""
import types

import numpy as np
import pytest

from tests.helpers import load
from tests.rerank_oracle import KS, STAGES, topk_ascending


@pytest.fixture(scope="module")
def z():
    return load("div_rerank.npz")


@pytest.mark.parametrize("stage", sorted(STAGES))
def test_fixture_is_the_top_k_of_the_reference_keys(z, stage):
    """Every stored pool is the top-k of the reference's own keys, in pool order; one document comes back squeezed."""
    Q = int(z["num_queries"])
    lens = [z[f"pool_{i}__docs"].shape[0] for i in range(Q)]
    assert min(lens) == 1 and max(lens) == 300 and Q >= 30
    for k in KS:
        for i in range(Q):
            docs, R, keys = z[f"pool_{i}__docs"], z[f"pool_{i}__rele"], z[f"{stage}__keys_{i}"]
            sel = topk_ascending(keys, k)
            if k > max(lens):
                assert f"{stage}_k{k}_{i}__docs" not in z.files
                continue
            got_d, got_R = z[f"{stage}_k{k}_{i}__docs"], z[f"{stage}_k{k}_{i}__rele"]
            if sel.size == 1:
                assert got_d.shape == (docs.shape[1],) and got_R.shape == (R.shape[0],)
            np.testing.assert_array_equal(got_d.reshape(sel.size, -1), docs[sel])
            np.testing.assert_array_equal(got_R.reshape(R.shape[0], sel.size), R[:, sel])


@pytest.mark.parametrize("stage", sorted(STAGES))
def test_fixture_keys_are_tie_free_at_every_cut(z, stage):
    for i in range(int(z["num_queries"])):
        keys = np.sort(z[f"{stage}__keys_{i}"].astype(np.float64))[::-1]
        span = max(keys[0] - keys[-1], 1e-6)
        for k in KS:
            if k < keys.size:
                assert keys[k - 1] - keys[k] > 1e-3 * span, (i, k)


def test_topk_restatement_orders_ties_by_index():
    keys = np.asarray([1.0, 3.0, 3.0, -0.0, 0.0, 3.0, 2.0], dtype=np.float32)
    np.testing.assert_array_equal(topk_ascending(keys, 2), [1, 2])
    np.testing.assert_array_equal(topk_ascending(keys, 4), [1, 2, 5, 6])
    np.testing.assert_array_equal(topk_ascending(keys, 6), [0, 1, 2, 3, 5, 6])
    np.testing.assert_array_equal(topk_ascending(keys, 9), np.arange(7))


def test_install_div_rerank_sets_only_the_dataset_class():
    import ptranking_b200
    from ptranking_b200.ltr_diversification.div_data import RerankDIVDataset
    old = object()
    module = types.SimpleNamespace(RerankDIVDataset=old, DIVDataset="div", DALETOR="d", DivProbRanker="p")
    before = dict(vars(module))
    previous = ptranking_b200.install_div_rerank(module)
    assert previous == {"RerankDIVDataset": old}
    assert module.RerankDIVDataset is RerankDIVDataset
    after = dict(vars(module))
    assert {k: v for k, v in after.items() if k != "RerankDIVDataset"} == \
        {k: v for k, v in before.items() if k != "RerankDIVDataset"}
    # install_diversification() leaves the dataset class alone
    module2 = types.SimpleNamespace(RerankDIVDataset=old)
    ptranking_b200.install_diversification(module2)
    assert module2.RerankDIVDataset is old


def test_rerank_k_below_one_is_refused():
    from ptranking_b200.ltr_diversification.div_data import RerankDIVDataset
    with pytest.raises(ValueError):
        RerankDIVDataset.from_queries([], discriminator=object(), rerank_k=0)
