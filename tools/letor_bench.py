"""Time read_letor on an MSLR-shaped file, stage by stage, on the GPU (CUDA events; the file read on the host clock).

    python tools/letor_bench.py [--lines 320000] [--repeats 3] [--out letor_bench.json]

The input is generated from a seed into a temporary directory: MSLR-WEB30K's shape (136 features, labels 0-4 with its
label mix, 20-240 documents per query), one line drawn per document from a pool of seeded feature rows.  Stages:
file read (host), host-to-device copy, line index + parse, grouping, and labels + clipping + scaling + presort +
gather, from the library's per-kernel event timing; and the whole call, file to device LetorSplit, on the host clock
after a synchronise.  A warm-up call precedes three timed repeats; the card's name and power limit are read in the
same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ptranking_b200 import _lib  # noqa: E402
from ptranking_b200.letor import read_letor  # noqa: E402

STAGES = {"index": ("count_newlines_kernel", "line_starts_kernel"),
          "parse": ("parse_lines_kernel",),
          "group": ("qid_insert_kernel", "first_flag_kernel", "line_query_kernel", "max_kernel", "scatter_lines_kernel",
                    "sort_query_lines_kernel"),
          "scale_clip_presort": ("query_labels_kernel", "shuffle_ties_kernel", "letor_gather_kernel")}
SCAN = ("scan_tile_sums_kernel", "scan_sums_kernel", "scan_apply_kernel")


def make_file(path, lines, seed=0, F=136):
    rng = np.random.default_rng(seed)
    pool = [" ".join("%d:%g" % (j + 1, v) for j, v in enumerate(np.round(rng.standard_normal(F) * 10 ** rng.integers(0, 4, F), 6)))
            for _ in range(2000)]
    written, q = 0, 0
    with open(path, "w") as f:
        while written < lines:
            n = min(int(rng.integers(20, 241)), lines - written)
            lab = rng.choice(5, n, p=[.515, .325, .134, .018, .008])
            rows = rng.integers(0, len(pool), n)
            f.write("".join(f"{lab[i]} qid:{q + 1} {pool[rows[i]]}\n" for i in range(n)))
            written += n
            q += 1
    return q


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    return r.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=320000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "letor_bench measures on a GPU"
    dd = dict(data_id="MSLRWEB30K", scale_data=True, scaler_id="StandardScaler", scaler_level="QUERY",
              min_docs=10, min_rele=1, binary_rele=False, unknown_as_zero=False)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "mslr.txt")
        nq = make_file(path, a.lines)
        nbytes = os.path.getsize(path)
        read_letor(path, dd, presort=True, seed=0)                              # warm-up
        torch.cuda.synchronize()
        runs = []
        for rep in range(a.repeats):
            t = time.perf_counter()
            with open(path, "rb") as f:
                f.read()
            t_read = time.perf_counter() - t
            host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
            with open(path, "rb") as f:
                f.readinto(memoryview(host.numpy()))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dev = host.to("cuda", non_blocking=True)
            e1.record()
            torch.cuda.synchronize()
            h2d = e0.elapsed_time(e1)
            del dev, host
            _lib.kernel_timings(True)
            torch.cuda.synchronize()
            t = time.perf_counter()
            sp = read_letor(path, dd, presort=True, seed=rep)
            torch.cuda.synchronize()
            total = time.perf_counter() - t
            _lib.kernel_timings(False)
            k = _lib.kernel_timings()
            stage = {s: sum(k.get(n, (0, 0.0))[1] for n in names) for s, names in STAGES.items()}
            stage["scans"] = sum(k.get(n, (0, 0.0))[1] for n in SCAN)
            runs.append(dict(file_read_ms=t_read * 1e3, h2d_ms=h2d, total_ms=total * 1e3, **{f"{s}_ms": v for s, v in stage.items()},
                             queries=len(sp), docs=int(sp.offsets_host[-1]), host_tokens=sp.host_tokens))
        res = dict(card=card(), lines=a.lines, bytes=nbytes, queries_in_file=nq, runs=runs,
                   MB_per_s=[nbytes / 1e6 / (r["total_ms"] / 1e3) for r in runs],
                   lines_per_s=[a.lines / (r["total_ms"] / 1e3) for r in runs])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
