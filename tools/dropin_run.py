"""The actual drop-in, end to end: the UNMODIFIED reference driver (ptranking.ltr_adhoc.eval.ltr.LTREvaluator.run,
ltr.py:568 -> point_run -> kfold_cv_eval :291-369) constructs, trains, validates, checkpoints, reloads and tests the
ptranking_b200 classes that ptranking_b200.install() registered in its module globals (ltr.py:166-171).

    python tools/dropin_run.py --impl b200 --model LambdaRank [--sf pointsf|listsf]      # on an H100
    python tools/dropin_run.py --impl reference --cuda none --model LambdaRank           # the reference itself, CPU

The reference is imported from baseline/_ref (a pip --target install of wildltr/ptranking, DESIGN.md section 8) or from
the checkout named by PTRANKING_REFERENCE.  Data: synthetic
LETOR-format files shaped like MSLR-WEB30K (136 features, grades 0-4 with the dataset's marginals, features weakly
informative so that learning shows) written to a scratch directory in the layout the loader expects
(<dir>/Fold{k}/{train,vali,test}.txt, ptranking/data/data_utils.py:553-640).  debug=True: 2 folds x 5 epochs, nDCG@5 validation.
"""
import argparse
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
import torch

P = np.array([1940952, 1225770, 504958, 69010, 30435], dtype=np.float64)
P /= P.sum()


def write_letor(path, rng, num_queries, qid0, F=136):
    w = rng.standard_normal(F) * (rng.random(F) < 0.2)            # a sparse linear relevance signal
    with open(path, "w") as f:
        for q in range(num_queries):
            n = int(rng.choice([40, 64, 100]))
            y = rng.choice(5, size=n, p=P)
            if y.max() < 1:
                y[rng.integers(n)] = 1
            X = rng.standard_normal((n, F)) * np.exp(rng.standard_normal(F) * 0.5) + 3.0 * rng.standard_normal(F)
            X += 0.35 * y[:, None] * w[None, :]
            for i in range(n):
                feats = " ".join(f"{k + 1}:{X[i, k]:.6f}" for k in range(F))
                f.write(f"{int(y[i])} qid:{qid0 + q} {feats}\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--cuda", default="0")
    ap.add_argument("--model", default="LambdaRank")
    ap.add_argument("--sf", default="pointsf", choices=["pointsf", "listsf"])
    ap.add_argument("--queries", type=int, default=240)
    ap.add_argument("--keep", action="store_true")
    ap.add_argument("--gpu-letor", action="store_true",
                    help="read the LETOR files on the device: ptranking_b200.install_data() replaces the driver's LTRDataset")
    args = ap.parse_args()

    work = tempfile.mkdtemp(prefix="dropin_")
    data_dir = os.path.join(work, "MSLRWEB30K") + "/"
    out_dir = os.path.join(work, "out") + "/"
    os.makedirs(out_dir)
    rng = np.random.default_rng(137)
    for fold in (1, 2):
        d = os.path.join(data_dir, f"Fold{fold}")
        os.makedirs(d)
        write_letor(os.path.join(d, "train.txt"), rng, args.queries, 10000 * fold)
        write_letor(os.path.join(d, "vali.txt"), rng, args.queries // 4, 10000 * fold + 4000)
        write_letor(os.path.join(d, "test.txt"), rng, args.queries // 4, 10000 * fold + 8000)

    import ptranking.ltr_adhoc.eval.ltr as ref_ltr
    from ptranking.ltr_adhoc.eval.ltr import LTREvaluator
    print(f"reference imported from {REF}; impl = {args.impl}; model = {args.model}; scorer = {args.sf}")
    if args.impl == "b200":
        import ptranking_b200
        prev = ptranking_b200.install()
        cls = getattr(ref_ltr, args.model)
        assert cls.__module__.startswith("ptranking_b200"), cls
        print(f"installed: ptranking.ltr_adhoc.eval.ltr.{args.model} -> {cls.__module__}.{cls.__name__}")
    if args.gpu_letor:
        import ptranking_b200
        ptranking_b200.install_data()
        print(f"installed: ptranking.ltr_adhoc.eval.ltr.LTRDataset -> {ref_ltr.LTRDataset.__module__}.LTRDataset")
    cuda = None if args.cuda == "none" else int(args.cuda)
    evaluator = LTREvaluator(cuda=cuda)
    t0 = time.time()
    evaluator.run(debug=True, model_id=args.model, sf_id=args.sf, data_id="MSLRWEB30K", dir_data=data_dir, dir_output=out_dir)
    dt = time.time() - t0
    print(f"LTREvaluator.run finished in {dt:.1f} s (2 folds x 5 epochs, {args.queries} train queries per fold)")
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
