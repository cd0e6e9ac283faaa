"""The diversification drop-in, end to end: the UNMODIFIED reference driver
(ptranking.ltr_diversification.eval.ltr_diversification.DivLTREvaluator.run -> point_run -> div_cv_eval, :304-375)
constructs, trains, validates, checkpoints, reloads and tests the DALETOR class that
ptranking_b200.install_diversification() registered in its module globals (:385-389).

    python tools/div_dropin_run.py --impl b200                      # on an H100
    python tools/div_dropin_run.py --impl reference --cuda none     # the reference itself, CPU

The reference is imported from baseline/_ref (a pip --target install of wildltr/ptranking, DESIGN.md section 8) or from
the checkout named by PTRANKING_REFERENCE.  Data: a synthetic data directory in the TREC Web-track diversification
layout the driver reads (load_raw_data, :155-207) -- query_permutation.json, query_representation.dat,
doc_representation.dat, query_doc.json and folder{1..5}/config.yml -- with 100-dimensional representations and
documents covering 1 to 6 subtopics.  debug=True (5 folds, alpha-nDCG@5 validation), 2 epochs, the pointsf scorer
by default; ``--sf listsf`` runs the list scorer with the reference's default listsf dict (div_parameter.py:98-104).

``--model DivProbRanker`` trains DivProbRanker instead.  ``--gpu-data`` (with ``--impl b200``) builds the plain splits
with the device DIVDataset through ptranking_b200.install_div_data().

``--rerank`` runs rerank mode end to end (ltr_diversification.py:323-335, util/div_data.py:130-192): the driver first
trains a DivProbRanker first stage (scorer ``--sf``), whose per-fold checkpoints stay where the driver wrote them
(<dir_run>/Fold-k/, the layout load_pretrained_model and get_opt_model read); the tool writes the rerank_dir JSONs
that describe it, and the driver then trains and tests DALETOR and DivProbRanker with both scorers on the pools the
first stage selects (rerank_k = RERANK_K), with ptranking_b200.install_div_rerank() in place for ``--impl b200``.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
for cand in (os.path.join(ROOT, "baseline", "_ref"), os.environ.get("PTRANKING_REFERENCE", "")):
    if os.path.isdir(os.path.join(cand, "ptranking")):
        sys.path.insert(0, cand)
        REF = cand
        break
else:
    raise SystemExit("the reference package is not available (baseline/_ref missing)")

import numpy as np

# the reference's load_raw_data uses np.float, which numpy 1.24 removed
np.float = float

EPOCHS = 2
RERANK_K = 20


def write_div_data(root, rng, queries_per_fold=12, F=100):
    """Representations: each query has a few latent subtopic directions; a document covering subtopic t lies near
    direction t, so the relevance is learnable from [q, q*d, d]."""
    perms, q_reprs, d_reprs, q_docs = {}, {}, {}, {}
    qid = 0
    folds = {}
    for fold in range(1, 6):
        folds[fold] = []
        for _ in range(queries_per_fold):
            qid += 1
            m = int(rng.integers(2, 7))
            dirs = rng.standard_normal((m, F))
            q = rng.standard_normal(F)
            q_reprs[str(qid)] = q.tolist()
            n = int(rng.integers(15, 60))
            docs, subtopics = [], {}
            for j in range(n):
                doc = f"q{qid}-d{j}"
                cover = [t + 1 for t in range(m) if rng.random() < 0.15]
                vec = rng.standard_normal(F) + sum(dirs[t - 1] for t in cover)
                d_reprs[doc] = vec.tolist()
                docs.append(doc)
                if cover:
                    subtopics[doc] = [str(t) for t in cover]
            if not subtopics:                       # every query has something to learn from
                subtopics[docs[0]] = ["1"]
            perms[str(qid)] = dict(alphaDCG=0.0, permutation=docs)
            q_docs[str(qid)] = subtopics
            folds[fold].append(qid)
    for name, obj in (("query_permutation.json", perms), ("query_representation.dat", q_reprs),
                      ("doc_representation.dat", d_reprs), ("query_doc.json", q_docs)):
        with open(os.path.join(root, name), "w") as f:
            json.dump(obj, f)
    for fold, qids in folds.items():
        os.makedirs(os.path.join(root, f"folder{fold}"))
        with open(os.path.join(root, f"folder{fold}", "config.yml"), "w") as f:
            f.write("test_set: [" + ", ".join(str(q) for q in qids) + "]\n")


def write_rerank_dir(rerank_dir, sf_para_dict, model_para_dict):
    """The first stage's scorer and model settings in the JSON layout get_rerank_para_dicts reads
    (DivScoringFunctionParameter / DivProbRankerParameter with para_json)."""
    sf_id = sf_para_dict["sf_id"]
    sf = sf_para_dict[sf_id]
    if sf_id == "pointsf":
        body = dict(layers=[sf["num_layers"]], AF=[sf["AF"]], apply_tl_af=[sf["apply_tl_af"]], TL_AF=[sf["TL_AF"]],
                    BN=[sf["BN"]], bn_type=[sf["bn_type"]], bn_affine=[sf["bn_affine"]])
    else:
        body = dict(BN=[sf["BN"]], bn_type=[sf["bn_type"]], bn_affine=[sf["bn_affine"]], ff_dims=sf["ff_dims"],
                    AF=[sf["AF"]], apply_tl_af=[sf["apply_tl_af"]], TL_AF=[sf["TL_AF"]], n_heads=[sf["n_heads"]],
                    encoder_type=[sf["encoder_type"]], encoder_layers=[sf["encoder_layers"]])
    sf_json = {"DivSFParameter": {"sf_id": sf_id, "opt": [sf_para_dict["opt"]], "lr": [sf_para_dict["lr"]], sf_id: body}}
    with open(os.path.join(rerank_dir, "Div_Data_Eval_ScoringFunction.json"), "w") as f:
        json.dump(sf_json, f)
    with open(os.path.join(rerank_dir, "DivProbRankerParameter.json"), "w") as f:
        json.dump({k: [v] for k, v in model_para_dict.items() if k != "model_id"}, f)


def run_rerank(args, ref_div, DivEvalSetting, data_dir, out_dir, work):
    """First stage, then the four second-stage runs; returns the number of runs that finished."""
    import torch
    debug_setting = DivEvalSetting.default_setting
    rerank = {}

    def with_rerank(self):
        d = debug_setting(self)
        d.update(rerank)
        return d
    DivEvalSetting.default_setting = with_rerank
    cuda = None if args.cuda == "none" else int(args.cuda)

    torch.manual_seed(2021)
    first = ref_div.DivLTREvaluator(cuda=cuda)
    t0 = time.time()
    first.run(debug=True, model_id="DivProbRanker", sf_id=args.sf, data_id="WT_Div_0912_Implicit", dir_data=data_dir,
              dir_output=os.path.join(out_dir, "first_stage") + "/")
    model_dir = first.dir_run
    folds = sorted(os.listdir(model_dir))
    print(f"first stage DivProbRanker ({args.sf}) trained in {time.time() - t0:.1f} s; checkpoints: "
          + ", ".join(f"{fd}/{os.listdir(os.path.join(model_dir, fd))}" for fd in folds if fd.startswith("Fold-")))
    rerank_dir = os.path.join(work, "rerank_cfg") + "/"
    os.makedirs(rerank_dir)
    write_rerank_dir(rerank_dir, first.sf_parameter.sf_para_dict, first.model_parameter.probrank_para_dict)
    rerank.update(rerank=True, rerank_k=RERANK_K, rerank_dir=rerank_dir, rerank_model_id="DivProbRanker",
                  rerank_model_dir=model_dir)
    done = 0
    for model_id in ("DALETOR", "DivProbRanker"):
        for sf_id in ("pointsf", "listsf"):
            torch.manual_seed(2021)
            ev = ref_div.DivLTREvaluator(cuda=cuda)
            print(f"== rerank mode: {model_id} ({sf_id}) on the top {RERANK_K} of the first stage")
            t0 = time.time()
            ev.run(debug=True, model_id=model_id, sf_id=sf_id, data_id="WT_Div_0912_Implicit", dir_data=data_dir,
                   dir_output=os.path.join(out_dir, f"rerank_{model_id}_{sf_id}") + "/")
            print(f"== {model_id} ({sf_id}) finished in {time.time() - t0:.1f} s (5 folds x {EPOCHS} epochs)")
            done += 1
    return done


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--cuda", default="0")
    ap.add_argument("--keep", action="store_true")
    ap.add_argument("--sf", default="pointsf", choices=["pointsf", "listsf"])
    ap.add_argument("--model", default="DALETOR", choices=["DALETOR", "DivProbRanker"])
    ap.add_argument("--rerank", action="store_true")
    ap.add_argument("--gpu-data", action="store_true",
                    help="build the plain splits with the device DIVDataset (ptranking_b200.install_div_data())")
    args = ap.parse_args()

    work = tempfile.mkdtemp(prefix="div_dropin_")
    data_dir = os.path.join(work, "WT_Div_0912_Implicit") + "/"
    out_dir = os.path.join(work, "out") + "/"
    os.makedirs(data_dir)
    os.makedirs(out_dir)
    write_div_data(data_dir, np.random.default_rng(2021))

    import torch
    import ptranking.ltr_diversification.eval.ltr_diversification as ref_div
    from ptranking.ltr_diversification.eval.div_parameter import DivEvalSetting
    print(f"reference imported from {REF}; impl = {args.impl}; model = {args.model}; scorer = {args.sf}; "
          f"rerank = {args.rerank}; device DIVDataset = {args.gpu_data}")
    if args.impl == "b200":
        import ptranking_b200
        ptranking_b200.install_diversification()
        assert ref_div.DALETOR.__module__.startswith("ptranking_b200"), ref_div.DALETOR
        print(f"installed: {ref_div.__name__}.DALETOR -> {ref_div.DALETOR.__module__}.DALETOR")
        if args.rerank:
            ptranking_b200.install_div_rerank()
            print(f"installed: {ref_div.__name__}.RerankDIVDataset -> {ref_div.RerankDIVDataset.__module__}")
        if args.gpu_data:
            ptranking_b200.install_div_data()
            print(f"installed: {ref_div.__name__}.DIVDataset -> {ref_div.DIVDataset.__module__}")

    # debug=True trains 5 epochs per fold; keep the run short without touching the driver
    debug_setting = DivEvalSetting.default_setting

    def two_epochs(self):
        d = debug_setting(self)
        d["epochs"] = EPOCHS
        return d
    DivEvalSetting.default_setting = two_epochs

    if args.rerank:
        done = run_rerank(args, ref_div, DivEvalSetting, data_dir, out_dir, work)
        print(f"rerank mode: {done} of 4 second-stage runs finished")
    else:
        torch.manual_seed(2021)
        cuda = None if args.cuda == "none" else int(args.cuda)
        evaluator = ref_div.DivLTREvaluator(cuda=cuda)
        t0 = time.time()
        evaluator.run(debug=True, model_id=args.model, sf_id=args.sf, data_id="WT_Div_0912_Implicit",
                      dir_data=data_dir, dir_output=out_dir)
        dt = time.time() - t0
        print(f"DivLTREvaluator.run finished in {dt:.1f} s (5 folds x {EPOCHS} epochs)")
    if args.impl == "b200":
        from ptranking_b200 import _lib
        print(f"kernels launched by libptranking_b200.so in this process: {_lib.launch_count()}")
        assert _lib.launch_count() > 0
    ckpts = [os.path.join(r, f) for r, _, fs in os.walk(out_dir) for f in fs if f.endswith(".pkl")]
    print(f"checkpoints written by the driver: {len(ckpts)}")
    if not args.keep:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
