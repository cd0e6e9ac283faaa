"""GPU parity of DALETOR with the diversification list scorer (sf_id='listsf'): the list-order feature, pitched padding
and concat kernels against torch indexing; the whole ranker against the unmodified reference's outputs
(tests/golden/divlist.npz) and the CPU oracle of tests/divlist_oracle.py, at head widths 10, 30, 50 and 150 (none a
multiple of 4, so every attention contraction takes the shape-general kernel); ragged steps, chunked split evaluation,
checkpoints and an evaluator-shaped run."""
import copy

import numpy as np
import pytest
import torch

from tests import daletor_oracle as do
from tests import divlist_oracle as dl
from tests.helpers import load, rel_err
from tests.test_oracle_divlist import SMALL, case_config, case_queries, final_checks

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# the JSON of the reference's diversification test setup (Div_Data_Eval_ScoringFunction.json)
JSON_LISTSF = dict(encoder_type="DASALC", encoder_layers=3, n_heads=2, BN=True, bn_type="BN", bn_affine=True,
                   ff_dims=[128, 256, 512], apply_tl_af=False, AF="R")


def _ranker(F, cfg, seeded=True, opt="Adagrad", lr=0.01):
    from ptranking_b200 import DALETOR
    sf = dict(sf_id="listsf", opt=opt, lr=lr, listsf=dict(num_features=F, **copy.deepcopy(cfg)))
    r = DALETOR(sf_para_dict=sf, model_para_dict=dict(model_id="DALETOR", rt=10.0, top_k=10), gpu=True, device=DEV)
    r.init()
    if seeded:
        init = dl.seeded_state(dl.state_shapes(r.list_sf["encoder"], r.list_sf["uni_sf"]))
        with torch.no_grad():
            for part in ("encoder", "uni_sf"):
                for k, v in r.list_sf[part].state_dict().items():
                    v.copy_(torch.from_numpy(init[part][k]))
    return r


def _pre_bn_bias(part, key, cfg):
    """uni_sf Linear biases that feed a BN: exactly 0 gradient from the per-query BN kernels (DESIGN §2)."""
    last = len(cfg["ff_dims"]) + 2
    return part == "uni_sf" and cfg.get("BN", True) and key.startswith("ff_") and key.endswith(".bias") \
        and key != f"ff_{last}.bias"


def _named_grads(r):
    return {(part, k): p.grad.detach().cpu().numpy() for part in ("encoder", "uni_sf")
            for k, p in r.list_sf[part].named_parameters()}


def _check_grads(got, want, cfg, rel=3e-5):
    """Per entry within ``rel`` of the tensor's largest reference entry, plus 2e-6 of the step's largest entry."""
    gscale = max(float(np.abs(w).max()) for w in want.values())
    for (part, key), w in want.items():
        g = got[(part, key)]
        if _pre_bn_bias(part, key, cfg):
            assert np.abs(g).max() == 0.0, (part, key)
            continue
        err = float(np.abs(g - w).max())
        assert err <= rel * float(np.abs(w).max()) + 2e-6 * gscale + 1e-9, (part, key, err, float(np.abs(w).max()), gscale)


# ---- kernels ------------------------------------------------------------------------------------------------------ #
def test_div_list_features_dense_and_ragged():
    from ptranking_b200 import ops
    rng = np.random.default_rng(9)
    F, lens = 20, [5, 0, 17, 1]
    q = torch.from_numpy(rng.standard_normal((4, F)).astype(np.float32))
    d = torch.from_numpy(rng.standard_normal((sum(lens), F)).astype(np.float32))
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
    X = ops.div_list_features(q.to(DEV), d.to(DEV), offsets=off, max_len=max(lens)).cpu()
    o = np.concatenate([[0], np.cumsum(lens)])
    for i in range(4):
        dq = d[o[i]:o[i + 1]]
        want = torch.cat((q[i:i + 1].expand(dq.size(0), -1), dq, q[i:i + 1] * dq), 1)    # div_list_ranker.py:62-64
        assert torch.equal(X[o[i]:o[i + 1]], want)
    Xd = ops.div_list_features(q[:1].to(DEV), d[:5].unsqueeze(0).to(DEV)).cpu()
    assert torch.equal(Xd[0], X[:5])


def _ragged(rng, lens, C):
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
    return off, torch.from_numpy(rng.standard_normal((sum(lens), C)).astype(np.float32)).to(DEV)


def test_pad_lists_pitched_and_concat_against_torch_indexing():
    from ptranking_b200 import ops
    rng = np.random.default_rng(3)
    lens, W = [7, 0, 130, 1, 64, 33], 150
    o = np.concatenate([[0], np.cumsum(lens)])
    off, X = _ragged(rng, lens, W)
    classes = [([2, 4], 130), ([5, 0], 40), ([3], 1)]       # any query order, a class longer than its lists
    qidxs = [torch.tensor(qs, dtype=torch.int32, device=DEV) for qs, _ in classes]
    # padding a column block of wider rows
    G = torch.from_numpy(rng.standard_normal((sum(lens), 2 * W)).astype(np.float32)).to(DEV)
    for (qs, n), qi in zip(classes, qidxs):
        for src, c0 in ((X, 0), (G, W)):
            P = ops.pad_lists_pitched(src, off, qi, n, col0=c0, width=W)
            want = torch.zeros(len(qs), n, W, device=DEV)
            for b, q in enumerate(qs):
                want[b, :lens[q]] = src[o[q]:o[q + 1], c0:c0 + W]
            assert torch.equal(P, want)
    # the concat: forward against torch.cat, backward exact zeros behind every list
    blocks = [torch.from_numpy(rng.standard_normal((len(qs), n, W)).astype(np.float32)).to(DEV).requires_grad_(True)
              for qs, n in classes]
    Z = ops.div_list_concat(X, off, qidxs, blocks)
    want = torch.zeros(sum(lens), 2 * W, device=DEV)
    want[:, :W] = X
    for (qs, n), blk in zip(classes, blocks):
        for b, q in enumerate(qs):
            want[o[q]:o[q + 1], W:] = blk[b, :lens[q]].detach()
    assert torch.equal(Z, want)
    (Z * G).sum().backward()
    for (qs, n), blk in zip(classes, blocks):
        for b, q in enumerate(qs):
            assert torch.equal(blk.grad[b, :lens[q]], G[o[q]:o[q + 1], W:])
            assert (blk.grad[b, lens[q]:] == 0).all()                       # exact zeros at padding


def test_new_entry_points_reject_bad_arguments():
    from ptranking_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(8, device=DEV)
    p = x.data_ptr()
    assert lib.ptrb200_div_list_features(p, p, None, p, 0, 4, 2, None) != 0             # B = 0
    assert lib.ptrb200_div_list_features(None, p, None, p, 1, 4, 2, None) != 0
    assert lib.ptrb200_pad_lists_pitched(p, 1, p, None, p, 1, 4, 2, None) != 0          # ld_src < W
    assert lib.ptrb200_pad_lists_pitched(p, 2, None, None, p, 1, 4, 2, None) != 0       # no offsets
    assert lib.ptrb200_div_list_concat(p, None, p, None, p, 1, 4, 2, None) != 0         # no encoder block
    assert lib.ptrb200_div_list_concat(p, p, p, None, p, 1, 0, 2, None) != 0            # n_max = 0
    assert b"div_list_concat" in lib.ptrb200_last_error()


# ---- the ranker against the reference's fixtures --------------------------------------------------------------------- #
def _train_op(r, q, d, R):
    return r.div_train_op(torch.from_numpy(q), torch.from_numpy(d), torch.from_numpy(R), presort=True, epoch_k=1)


@pytest.mark.parametrize("name", SMALL + ["default"])
def test_ranker_matches_reference_fixture(name):
    z = load("divlist.npz")
    F, cfg = case_config(name)
    qs = case_queries(name)
    r = _ranker(F, cfg)
    r.eval_mode()
    with torch.no_grad():
        for i, (q, d, _) in enumerate(qs):
            got = r.div_forward(torch.from_numpy(q).to(DEV), torch.from_numpy(d).to(DEV)).cpu().numpy()
            assert rel_err(got, z[f"{name}__pred_q{i}"]) <= 2e-5, (i, rel_err(got, z[f"{name}__pred_q{i}"]))
    for i, (q, d, R) in enumerate(qs):              # one DALETOR step of each query from the starting weights
        r = _ranker(F, cfg)
        r.eval_mode()
        loss, stop = _train_op(r, q, d, R)
        want = float(z[f"{name}__loss_q{i}"])
        assert not stop and abs(float(loss.detach()) - want) <= 3e-5 * max(1.0, abs(want)), (i, float(loss), want)
        if i == dl.grad_query(name):
            want_g = {(part, k): z[f"{name}__grad__{part}__{k}"] for part in ("encoder", "uni_sf")
                      for k, _ in r.list_sf[part].named_parameters()}
            _check_grads(_named_grads(r), want_g, cfg)
    r = _ranker(F, cfg)                             # three Adagrad steps in turn
    r.eval_mode()
    losses = [float(_train_op(r, q, d, R)[0].detach()) for q, d, R in qs]
    assert abs(losses[0] - z[f"{name}__losses"][0]) <= 3e-5 * max(1.0, abs(losses[0]))
    tol, compared = final_checks(name, qs)            # why these bars: tests/test_oracle_divlist.py
    assert np.allclose(losses, z[f"{name}__losses"], rtol=tol, atol=1e-6), (losses, z[f"{name}__losses"])
    with torch.no_grad():
        for i in compared:
            q, d, _ = qs[i]
            got = r.div_forward(torch.from_numpy(q).to(DEV), torch.from_numpy(d).to(DEV)).cpu().numpy()
            assert rel_err(got, z[f"{name}__final_q{i}"]) <= tol, (i, rel_err(got, z[f"{name}__final_q{i}"]))


@pytest.mark.parametrize("heads", [6, 2])
def test_default_configuration_against_cpu_oracle(heads):
    """The reference default at F = 100 (6 layers, head widths 50 and 150) on a 256-document list: scores, loss and
    every parameter gradient against the CPU oracle."""
    cfg = dict(dl.DEFAULT_LISTSF, n_heads=heads)
    rng = np.random.default_rng(heads)
    n, F = 256, 100
    q = rng.standard_normal((1, F)).astype(np.float32)
    d = rng.standard_normal((n, F)).astype(np.float32)
    R = (rng.random((5, n)) < 0.2).astype(np.float32)
    R[0, 0] = 1.0
    r = _ranker(F, cfg)
    r.eval_mode()
    net = dl.OracleDivList(F, heads, cfg["encoder_layers"], cfg["encoder_type"], cfg["ff_dims"], cfg["AF"],
                           cfg["TL_AF"], cfg["apply_tl_af"], cfg["BN"], cfg["bn_type"], cfg["bn_affine"]).eval()
    net.load_reference_state({k: v.cpu() for k, v in r.list_sf["encoder"].state_dict().items()},
                             {k: v.cpu() for k, v in r.list_sf["uni_sf"].state_dict().items()})
    s_ref = net(torch.from_numpy(q), torch.from_numpy(d))
    loss_ref = do.port_loss(s_ref, torch.from_numpy(R), 10.0, 10)
    loss_ref.backward()
    want = {dl.reference_key_of(k): p.grad.numpy() for k, p in net.named_parameters()}
    with torch.no_grad():
        s = r.div_forward(torch.from_numpy(q).to(DEV), torch.from_numpy(d).to(DEV)).cpu().numpy()
    assert rel_err(s, s_ref.detach().numpy()) <= 2e-5, rel_err(s, s_ref.detach().numpy())
    loss, _ = _train_op(r, q, d, R)
    assert abs(float(loss.detach()) - float(loss_ref)) <= 3e-5 * max(1.0, abs(float(loss_ref)))
    _check_grads(_named_grads(r), want, cfg, rel=5e-5)


# ---- ragged steps, split evaluation ---------------------------------------------------------------------------------- #
def _queries(rng, lens, F, ms=None):
    out = []
    for i, n in enumerate(lens):
        m = ms[i] if ms else 4
        R = (rng.random((m, n)) < 0.25).astype(np.float32)
        R[0, 0] = 1.0
        out.append((f"q{i}", torch.from_numpy(rng.standard_normal((1, F)).astype(np.float32)),
                    [f"d{j}" for j in range(n)], torch.from_numpy(rng.standard_normal((n, F)).astype(np.float32)),
                    None, None, torch.from_numpy(R)))
    return out


def _step_grads(r, sp, q0, q1, params):
    from ptranking_b200 import ops
    o = sp.offsets_host
    X = sp.X[int(o[q0]):int(o[q1])]
    plan = sp.plan(q0, q1, r)
    s = r.list_scores(X, plan)
    loss, _ = ops.daletor_loss(s, sp.rele.select(q0, q1), rt=10.0, top_k=10, offsets=plan.offsets, max_len=plan.max_len)
    return s.detach(), loss.detach(), torch.autograd.grad(loss, params)


def test_ragged_step_is_deterministic_and_equals_per_query_steps():
    F, lens = 100, [1, 2, 17, 300, 1025]
    cfg = dict(dl.DEFAULT_LISTSF, encoder_layers=2)
    r = _ranker(F, cfg)
    r.eval_mode()
    data = _queries(np.random.default_rng(1), lens, F)
    sp = r._split(data)
    params = r.get_parameters()
    s, loss, g = _step_grads(r, sp, 0, len(lens), params)
    assert len(sp.plan(0, len(lens), r).classes) == 5                     # every length its own class
    s2, loss2, g2 = _step_grads(r, sp, 0, len(lens), params)
    assert torch.equal(s, s2) and torch.equal(loss, loss2) and all(torch.equal(a, b) for a, b in zip(g, g2))
    o = sp.offsets_host
    tot = [torch.zeros_like(p) for p in params]
    losses = 0.0
    for i in range(len(lens)):
        si, li, gi = _step_grads(r, sp, i, i + 1, params)
        assert rel_err(s[o[i]:o[i + 1]].cpu().numpy(), si.cpu().numpy()) <= 1e-5, i
        losses += float(li)
        for t, x in zip(tot, gi):
            t += x
    assert abs(float(loss) - losses) <= 1e-5 * max(1.0, abs(losses))
    gscale = max(float(t.abs().max()) for t in tot)
    for t, x in zip(tot, g):
        assert float((t - x).abs().max()) <= 1e-5 * float(t.abs().max()) + 1e-6 * gscale


def test_split_evaluation_in_chunks_equals_per_query_scoring():
    F, heads = 20, 6
    cfg = dict(dl.SMALL_LISTSF, encoder_type="AllRank", n_heads=heads)
    r = _ranker(F, cfg)
    rng = np.random.default_rng(5)
    lens = [3, 64, 64, 200, 9, 130, 64, 1, 40, 63, 17, 200]
    data = _queries(rng, lens, F, ms=[3] * len(lens))
    data[4] = data[4][:6] + (torch.zeros(3, 9),)                            # a query without relevance
    r.attn_budget_bytes = 4 * heads * 64 * 64 * 2                           # two 64-document lists per chunk
    sp = r._split(data)
    plan = sp.plan(0, len(sp), r)
    assert len(plan.classes) >= 8 and max(len(c[0]) for c in plan.classes) == 2
    r.eval_mode()
    with torch.no_grad():
        preds = r.list_scores(sp.X, plan).cpu().numpy()
        per = [r.div_predict(q.to(DEV), dr.to(DEV)).cpu().numpy()[0] for _, q, _, dr, _, _, _ in data]
    o = sp.offsets_host
    for i, p in enumerate(per):
        assert rel_err(preds[o[i]:o[i + 1]], p) <= 1e-5, i
    ks = [1, 3, 5, 10, 20]
    ms = [do.port_metrics(p, R.numpy(), ks, 1.0) for p, (*_, R) in zip(per, data)]
    cnt0 = [i for i, (*_, R) in enumerate(data) if float(R.sum()) > 0]
    a, e, ne = r.srd_performance_at_ks(test_data=data, ks=ks, max_label=1.0)
    for j, got in enumerate((a, e, ne)):
        assert np.abs(got.numpy() - np.mean([ms[i][j] for i in cnt0], axis=0)).max() <= 2e-5


def test_save_load_round_trip(tmp_path):
    r = _ranker(20, dict(dl.SMALL_LISTSF, encoder_type="DASALC", n_heads=2), seeded=False)
    data = _queries(np.random.default_rng(2), [30, 7], 20)
    r.div_train(data, epoch_k=1)
    r.save(str(tmp_path) + "/", "m.pkl")
    ck = torch.load(str(tmp_path) + "/m.pkl", map_location="cpu")
    assert set(ck) == {"encoder", "uni_sf"}
    r2 = _ranker(20, dict(dl.SMALL_LISTSF, encoder_type="DASALC", n_heads=2), seeded=False)
    r2.load(str(tmp_path) + "/m.pkl")                    # no device=, as the evaluator reloads it
    for part in ("encoder", "uni_sf"):
        a, b = r.list_sf[part].state_dict(), r2.list_sf[part].state_dict()
        assert all(torch.equal(a[k], b[k]) for k in a)
    r.eval_mode(), r2.eval_mode()
    with torch.no_grad():
        for _, q, _, d, _, _, _ in data:
            assert torch.equal(r.div_predict(q.to(DEV), d.to(DEV)), r2.div_predict(q.to(DEV), d.to(DEV)))


@pytest.mark.parametrize("which", ["default", "json"])
def test_evaluator_shaped_run(which):
    """What DivLTREvaluator calls, with the reference's listsf dicts: div_train epochs (one query per step, and
    several), div_validation, srd_performance_at_ks on lists shorter than max(ks)."""
    F = 100
    cfg, opt = (dl.DEFAULT_LISTSF, "Adagrad") if which == "default" else (JSON_LISTSF, "Adam")
    r = _ranker(F, cfg, seeded=False, opt=opt, lr=0.01)
    rng = np.random.default_rng(8)
    train = _queries(rng, [50, 3, 120, 30, 8, 200], F)
    vali = _queries(rng, [40, 4, 60], F)
    for epoch in range(1, 3):
        loss, stop = r.div_train(train, epoch_k=epoch)
        assert not stop and np.isfinite(float(loss))
    r.queries_per_step = 3
    loss, stop = r.div_train(train, epoch_k=10)
    assert not stop and np.isfinite(float(loss))
    v = float(r.div_validation(vali_data=vali, vali_metric="aNDCG", k=5))
    v2 = float(r.div_validation(vali_data=vali, vali_metric="nERR-IA", k=5, max_label=1.0))
    assert v >= 0.0 and v2 >= 0.0 and np.isfinite([v, v2]).all()      # the ideal is the input order: may exceed 1
    a, e, ne = r.srd_performance_at_ks(test_data=vali, ks=[1, 3, 5, 10, 20, 50], max_label=1.0)
    assert a.shape == (6,) and np.isfinite(a.numpy()).all() and np.isfinite(ne.numpy()).all()
    r.eval_mode()
    with torch.no_grad():
        per = [r.div_predict(q.to(DEV), d.to(DEV)).cpu().numpy()[0] for _, q, _, d, _, _, _ in vali]
    want = np.mean([do.port_metrics(p, R.numpy(), [1, 3, 5, 10, 20, 50], 1.0)[0] for p, (*_, R) in zip(per, vali)],
                   axis=0)
    assert np.abs(a.numpy() - want).max() <= 2e-5
