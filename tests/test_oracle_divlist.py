"""Pin the CPU restatement of the diversification list scorer (tests/divlist_oracle.py) to outputs of the unmodified
reference (tests/golden/divlist.npz, made by tests/golden/make_golden_divlist.py), and check the listsf ranker's
settings, checkpoint keys, parameter order and length classes without a GPU."""
import numpy as np
import pytest
import torch

from oracle import ref_port as rp
from tests import daletor_oracle as do
from tests import divlist_oracle as dl
from tests.helpers import load, rel_err

SMALL = dl.SMALL
# Scores and losses after three Adagrad steps: Adagrad's first step moves every parameter by about lr * sign(g), so
# gradient entries at rounding level (e.g. the Linear biases ahead of a BN, exactly 0 in exact arithmetic) turn into
# lr-sized parameter differences between any two fp32 implementations.  The first step's scores, loss and gradients are
# held to 2e-5 / 3e-5; after the steps the small cases are held to FINAL_TOL, the default scorer -- whose 2.4 M
# parameters all move by about lr = 0.01, so that small but real gradient entries whose sign two implementations see
# differently move by 2 lr apart -- to DEFAULT_FINAL_TOL (two CPU implementations of the same operations end 2.2e-2 and
# 5.4e-2 apart on the 256- and 37-document lists; a check of the direction, not of the digits).
# A 2-document list is not compared after the steps in the default case: a per-query BN over two rows outputs +-1 by
# the sign of their difference, a discontinuous function of the weights.
FINAL_TOL = 2e-3
DEFAULT_FINAL_TOL = 1e-1


def final_checks(name, qs):
    """-> (bar, indices of the queries whose post-step scores are compared)."""
    if name == "default":
        return DEFAULT_FINAL_TOL, [i for i, (_, d, _) in enumerate(qs) if len(d) > 2]
    return FINAL_TOL, list(range(len(qs)))


def case_config(name):
    """-> (F, listsf dict) of a fixture case."""
    return dl.case_config(name)[:2]


def case_queries(name):
    """[(q_repr, doc_reprs, rele)] of a fixture case (rebuilt, not stored)."""
    return dl.case_inputs(name)


def oracle(name):
    """OracleDivList with the case's seeded starting weights, in eval mode."""
    F, cfg = case_config(name)
    net = dl.OracleDivList(F, cfg["n_heads"], cfg["encoder_layers"], cfg["encoder_type"], cfg["ff_dims"], cfg["AF"],
                           cfg["TL_AF"], cfg["apply_tl_af"], cfg["BN"], cfg["bn_type"], cfg["bn_affine"])
    shapes = {"encoder": {}, "uni_sf": {}}
    for k, v in net.state_dict().items():
        part, key = dl.reference_key_of(k)
        shapes[part][key] = tuple(v.shape)
    init = dl.seeded_state(shapes)
    net.load_reference_state(init["encoder"], init["uni_sf"])
    return net.eval()


def _scores(net, q, d):
    return net(torch.from_numpy(q), torch.from_numpy(d))


def _step(net, opt, q, d, R):
    opt.zero_grad()
    loss = do.port_loss(_scores(net, q, d), torch.from_numpy(R), 10.0, 10)
    loss.backward()
    opt.step()
    return float(loss.detach())


@pytest.mark.parametrize("name", SMALL + ["default"])
def test_oracle_matches_reference(name):
    z = load("divlist.npz")
    qs = case_queries(name)
    net = oracle(name)
    with torch.no_grad():
        for i, (q, d, _) in enumerate(qs):
            assert rel_err(_scores(net, q, d).numpy(), z[f"{name}__pred_q{i}"]) <= 2e-5, i
    for i, (q, d, R) in enumerate(qs):
        net = oracle(name)
        opt, _ = rp.make_optimizer(net.parameters(), "Adagrad", 0.01)
        loss = _step(net, opt, q, d, R)
        assert abs(loss - float(z[f"{name}__loss_q{i}"])) <= 2e-5 * max(1.0, abs(loss)), i
        if i != dl.grad_query(name):
            continue
        grads = {dl.reference_key_of(k): p.grad.numpy() for k, p in net.named_parameters()}
        gscale = max(float(np.abs(g).max()) for g in grads.values())
        for (part, key), g in grads.items():
            want = z[f"{name}__grad__{part}__{key}"]
            assert np.abs(g - want).max() <= 1e-5 * np.abs(want).max() + 1e-6 * gscale, (i, part, key)
    net = oracle(name)
    opt, _ = rp.make_optimizer(net.parameters(), "Adagrad", 0.01)
    losses = [_step(net, opt, q, d, R) for q, d, R in qs]
    assert abs(losses[0] - z[f"{name}__losses"][0]) <= 2e-5 * max(1.0, abs(losses[0]))
    tol, compared = final_checks(name, qs)
    assert np.allclose(losses, z[f"{name}__losses"], rtol=tol, atol=1e-6)
    with torch.no_grad():
        for i in compared:
            q, d, _ = qs[i]
            assert rel_err(_scores(net, q, d).numpy(), z[f"{name}__final_q{i}"]) <= tol, i


def test_fixture_covers_the_cases():
    z = load("divlist.npz")
    names = {k.split("__")[0] for k in z.files}
    assert names == set(SMALL) | {"default"}
    lens = sorted(d.shape[0] for n in SMALL for _, d, _ in case_queries(n))
    assert lens[0] == 2 and lens[-1] > 128
    grad_lens = {case_queries(n)[dl.grad_query(n)][1].shape[0] for n in SMALL}
    assert grad_lens == {150, 37} and all(z[f"{n}__pred_q{i}"].shape == (1, len(case_queries(n)[i][1]))
                                          for n in SMALL + ["default"] for i in range(3))
    for name in SMALL:            # head widths 6 and 18: not multiples of 4
        F, cfg = case_config(name)
        assert (3 * F // cfg["n_heads"]) % 4 == 2


def _sf(listsf):
    return dict(sf_id="listsf", opt="Adagrad", lr=0.01, listsf=listsf)


def _model():
    return dict(model_id="DALETOR", rt=10.0, top_k=10)


@pytest.mark.parametrize("gpu,device", [(True, "cuda:0"), (False, "cpu")])
def test_listsf_constructor_validation(gpu, device):
    from ptranking_b200 import DALETOR
    for bad in ({}, dict(encoder_type="Transformer"), dict(num_features=20, encoder_type=None)):
        with pytest.raises(NotImplementedError, match="list scorer"):
            DALETOR(sf_para_dict=_sf(dict(bad)), model_para_dict=_model(), gpu=gpu, device=device)
    with pytest.raises(NotImplementedError, match="list scorer"):
        DALETOR(sf_para_dict=_sf(dict(num_features=20, encoder_type="AttnDIN", BN=True, bn_type="BN2")),
                model_para_dict=_model(), gpu=gpu, device=device)
    good = _sf(dict(num_features=20, **dl.DEFAULT_LISTSF))
    if not gpu:
        with pytest.raises(RuntimeError):              # CUDA only, no CPU fallback
            DALETOR(sf_para_dict=good, model_para_dict=_model(), gpu=gpu, device=device)
    else:
        r = DALETOR(sf_para_dict=good, model_para_dict=_model(), gpu=gpu, device=device)
        assert good["listsf"]["num_features"] == 20       # the list scorer widens its own layers
        assert r.encoder_type == "AttnDIN" and r.queries_per_step == 1


def _parts(F, cfg):
    """The listsf modules as the ranker builds them, on the CPU (construction touches no device)."""
    from ptranking_b200.ltr_diversification.base.div_list_ranker import DivListNeuralRanker
    host = DivListNeuralRanker()
    host.device = "cpu"
    host.list_sf = host.ini_listsf(num_features=F, **cfg)
    return host


@pytest.mark.parametrize("name", SMALL)
def test_checkpoint_keys_are_the_references(name):
    z = load("divlist.npz")
    F, cfg = case_config(name)
    host = _parts(F, cfg)
    for part in ("encoder", "uni_sf"):
        want = [k.split("__")[3] for k in z.files if k.startswith(f"{name}__grad__{part}__")]
        assert sorted(host.list_sf[part].state_dict()) == sorted(want), part
        assert {k: tuple(v.shape) for k, v in host.list_sf[part].state_dict().items()} == \
            {k: z[f"{name}__grad__{part}__{k}"].shape for k in want}


def test_default_parameter_count_and_order():
    host = _parts(100, dl.DEFAULT_LISTSF)
    ps = host.list_parameters()
    enc, uni = list(host.list_sf["encoder"].parameters()), list(host.list_sf["uni_sf"].parameters())
    assert sum(p.numel() for p in ps) == 2366769                       # 6 * 361,800 + 195,969
    assert sum(p.numel() for p in enc) == 6 * 361800 and sum(p.numel() for p in uni) == 195969
    assert {id(p) for p in ps[:len(enc)]} == {id(p) for p in enc}      # the encoder first
    assert [id(p) for p in ps[len(enc):]] == [id(p) for p in uni]      # then uni_sf, in its own order
    mhsa = host.list_sf["encoder"].layers[0].mhsa
    i = [id(p) for p in ps].index(id(mhsa.w_q.weight))                 # projection weights side by side
    assert ps[i + 1] is mhsa.w_k.weight and ps[i + 2] is mhsa.w_v.weight
    assert host.list_sf["uni_sf"].bn_per_query and host.list_sf["uni_sf"].spec.dropout_p == 0.1


def test_length_classes():
    from ptranking_b200.ltr_diversification.base.div_list_ranker import length_classes
    lens = [1, 2, 17, 300, 1025, 0, 600, 300, 513]
    cls = length_classes(lens, 6, budget=1 << 40)
    assert [n for _, n in cls] == [1025, 300, 17, 2, 1]
    assert [sorted(q) for q, _ in cls] == [[4, 6, 8], [3, 7], [2], [1], [0]]
    covered = sorted(q for qs, _ in cls for q in qs)
    assert covered == [0, 1, 2, 3, 4, 6, 7, 8]                          # every non-empty query once
    for qs, n in cls:
        assert all(lens[q] <= n and 2 * lens[q] > n for q in qs)
    # a budget of two 300-document queries' attention tensors
    cls = length_classes([300] * 5, 6, budget=2 * 4 * 6 * 300 * 300)
    assert [len(q) for q, _ in cls] == [2, 2, 1]
    assert [len(q) for q, _ in length_classes([4096], 6, budget=1)] == [1]   # one list always goes, whatever the budget
