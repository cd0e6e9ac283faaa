"""Achieved parity errors on the GPU -> profiles/<tag>_parity_table.md (VERDICT r1 item 1e).

For every loss x n in {32, 256, 512, 1024} and every pointwise-scorer configuration: the error of the CUDA path against
(i) the oracle = the reference's own fp32 ATen ops on the CPU, (ii) float64 truth (closed forms for the losses, the oracle
network in double precision for the scorer), in three norms:
    maxabs  = max|a-b| / max|b|                 (what the tests assert)
    l2      = ||a-b||_2 / ||b||_2               (norm-wise)
    elem    = max_i |a_i-b_i| / max(|b_i|, 1e-4 max|b|)   (element-wise, floored where the reference is ~0)
The column "ref vs f64" is the fp32 reference's own distance from float64 -- the rounding noise no fp32 kernel can beat.
    python tools/parity_table.py [tag]
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from oracle import closed_form as cf
from oracle import ref_port as rp
from ptranking_b200 import ops

tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
dev = "cuda:0"
P = np.array([1940952, 1225770, 504958, 69010, 30435], dtype=np.float64); P /= P.sum()


def errs(a, b):
    a = np.asarray(a, dtype=np.float64).reshape(-1); b = np.asarray(b, dtype=np.float64).reshape(-1)
    mb = max(np.abs(b).max(), 1e-300)
    return (np.abs(a - b).max() / mb, np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300),
            (np.abs(a - b) / np.maximum(np.abs(b), 1e-4 * mb)).max())


def fmt(e):
    return " / ".join(f"{x:.1e}" for x in e)


def synth(B, n, seed):
    rng = np.random.default_rng(seed)
    y = rng.choice(5, size=(B, n), p=P).astype(np.float32)
    y[:, 0] = np.maximum(y[:, 0], 1.0)
    y = -np.sort(-y, axis=1)
    s = (1.0 / (1.0 + np.exp(-rng.standard_normal((B, n))))).astype(np.float32)       # scorer outputs after the sigmoid tail
    return s, y


LOSSES = [("RankNet", dict(sigma=1.0)), ("LambdaRank", dict(sigma=1.0)),
          ("LambdaLoss", dict(k=5, sigma=1.0, mu=5.0, loss_type="NDCG_Loss2++", presort=True)),
          ("LambdaLoss", dict(k=10 ** 6, sigma=1.0, mu=5.0, loss_type="NDCG_Loss2++", presort=True)),
          ("ListNet", {}), ("ListMLE", {}), ("ApproxNDCG", dict(alpha=10.0, presort=True)),
          ("RankMSE", {}), ("RankCosine", {}), ("STListNet", dict(temperature=1.0)), ("SoftRank", dict(delta=2.0, top_k=None))]


def closed(name, s, y, params, extra):
    p = {k: v for k, v in params.items() if k != "presort"}
    if name == "RankNet": return cf.ranknet(s, y, **p)
    if name == "LambdaRank": return cf.lambdarank(s, y, **p)
    if name == "LambdaLoss": return cf.lambdaloss(s, y, presort=True, **{**p, "k": min(p["k"], s.shape[1])})
    if name == "ListNet": return cf.listnet(s, y)
    if name == "ListMLE": return cf.listmle(s, extra["perm"])
    if name == "ApproxNDCG": return cf.approxndcg(s, y, presort=True, **p)
    if name == "RankMSE": return cf.rankmse(s, y)
    if name == "RankCosine": return cf.rankcosine(s, y)
    if name == "STListNet": return cf.stlistnet(s, y, extra["unif"], **p)
    return cf.softrank(s, y, **p)


lines = []
lines.append("| loss | n | grad: CUDA vs reference fp32 | grad: CUDA vs float64 | grad: ref fp32 vs float64 | loss rel: vs ref / vs f64 / ref vs f64 |")
lines.append("|---|---|---|---|---|---|")
worst = 0.0
for name, params in LOSSES:
    for n in (32, 256, 512, 1024):
        B = 8
        s, y = synth(B, n, seed=n + len(name))
        kw, okw, extra = dict(params), dict(params), {}
        if name == "LambdaLoss":
            kw["k"] = okw["k"] = min(params["k"], n)
        if name == "ListMLE":
            perm = rp.shuffle_ties_perm(torch.from_numpy(y), generator=torch.Generator().manual_seed(n))
            extra["perm"] = perm.numpy(); kw["perm"] = perm.to(torch.int32).to(dev); okw["perm"] = perm
        if name == "STListNet":
            u = torch.rand(B, n, generator=torch.Generator().manual_seed(n))
            extra["unif"] = u.numpy(); kw["unif"] = u.to(dev); okw["unif"] = u
        loss, _, grad = ops.rank_loss_and_grad(name, torch.from_numpy(s).to(dev), torch.from_numpy(y).to(dev), **kw)
        loss, grad = float(loss), grad.cpu().numpy()
        ol, og = rp.loss_and_grad(name, torch.from_numpy(s), torch.from_numpy(y), **okw)
        ol, og = float(ol), og.numpy()
        fl, fg = closed(name, s, y, okw if name == "LambdaLoss" else params, extra)
        e_ref, e_f64, r_f64 = errs(grad, og), errs(grad, fg), errs(og, fg)
        worst = max(worst, e_f64[0])
        lab = name + (f" {params.get('loss_type')} k={'n' if params['k'] > 10 ** 5 else params['k']}" if name == "LambdaLoss" else "")
        lines.append(f"| {lab} | {n} | {fmt(e_ref)} | {fmt(e_f64)} | {fmt(r_f64)} | "
                     f"{abs(loss - ol) / max(abs(ol), 1e-30):.1e} / {abs(loss - fl) / max(abs(fl), 1e-30):.1e} / {abs(ol - fl) / max(abs(fl), 1e-30):.1e} |")

# ---- scorers ---------------------------------------------------------------------------------
import ptranking_b200
from tests.test_oracle_vs_golden import POINT_CFGS, point_cfg

slines = ["| scorer config | shape | scores: vs ref fp32 | scores: vs float64 | ref vs float64 | worst param grad: vs ref fp32 | vs float64 | ref vs float64 |",
          "|---|---|---|---|---|---|---|---|"]
cfgs = dict(POINT_CFGS)
for code in ("T", "E", "LR", "SE"):
    cfgs["af_" + code] = dict(AF=code, TL_AF=code, num_layers=3)
for name, over in cfgs.items():
    for (B, n, F) in [(4, 64, 136), (64, 256, 136)] if name == "default" else [(4, 64, 136)]:
        torch.manual_seed(11)
        sf = dict(sf_id="pointsf", opt="Adam", lr=1e-4, pointsf=point_cfg(F, **over))
        r = ptranking_b200.ListNet(sf_para_dict=sf, gpu=True, device=dev)
        r.init(); r.eval_mode()
        net = rp.point_scorer(**sf["pointsf"])
        net.load_state_dict({k: v.cpu() for k, v in r.point_sf.state_dict().items()})
        net.eval()
        import copy
        net64 = copy.deepcopy(net).double()
        g = torch.Generator().manual_seed(3)
        X = torch.randn(B, n, F, generator=g); w = torch.randn(B, n, generator=g)
        s = r.forward(X.to(dev)); r.grad_bucket.zero(); (s * w.to(dev)).sum().backward()
        s32 = rp.point_forward(net, X); (s32 * w).sum().backward()
        s64 = rp.point_forward(net64, X.double()); (s64 * w.double()).sum().backward()
        es = (errs(s.detach().cpu().numpy(), s32.detach().numpy()), errs(s.detach().cpu().numpy(), s64.detach().numpy()),
              errs(s32.detach().numpy(), s64.detach().numpy()))
        gs = max(np.abs(p.grad.numpy()).max() for p in net64.parameters())
        wg = [0.0, 0.0, 0.0]
        for (k, p), p32, p64 in zip(r.point_sf.named_parameters(), net.parameters(), net64.parameters()):
            a, b32, b64 = p.grad.cpu().numpy().astype(np.float64), p32.grad.numpy().astype(np.float64), p64.grad.numpy()
            # relative to the net's gradient scale: biases feeding a norm have exactly-zero true gradients
            wg[0] = max(wg[0], np.abs(a - b32).max() / gs); wg[1] = max(wg[1], np.abs(a - b64).max() / gs); wg[2] = max(wg[2], np.abs(b32 - b64).max() / gs)
        slines.append(f"| {name} | {B}x{n}x{F} | {fmt(es[0])} | {fmt(es[1])} | {fmt(es[2])} | {wg[0]:.1e} | {wg[1]:.1e} | {wg[2]:.1e} |")

os.makedirs("profiles", exist_ok=True)
with open(f"profiles/{tag}_parity_table.md", "w") as f:
    f.write(f"# {tag}: achieved parity errors on one {torch.cuda.get_device_name()} (`python tools/parity_table.py`, through the C ABI)\n\n")
    f.write("Three numbers per cell: maxabs / l2 / elem (definitions in the tool's docstring).  B = 8 queries per loss case; scores are\n"
            "sigmoid outputs (the default scorer's tail), labels follow the MSLR-WEB30K marginals, presorted.  north_star's bar: loss and\n"
            "gradient within 1e-5 relative fp32 of the reference; where the reference itself sits further than that from float64\n"
            "(long fp32 sums at n >= 512) the kernel is held to the float64 truth instead.\n\n")
    f.write("## losses\n\n" + "\n".join(lines) + "\n\n")
    f.write(f"worst gradient maxabs error against float64 over all loss cases: {worst:.2e}\n\n")
    f.write("## pointwise scorer (forward scores and parameter gradients of sum(scores * w), dropout off)\n\n" + "\n".join(slines) + "\n\n")
    f.write("Parameter-gradient errors are relative to the largest gradient entry of the net (a Linear bias feeding a normalisation has an\n"
            "exactly-zero true gradient; both fp32 sides hold rounding noise there).\n")
print(open(f"profiles/{tag}_parity_table.md").read())
