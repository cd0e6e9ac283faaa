"""Writes tests/golden/letor.npz: small seeded LETOR files and what the reference's loader makes of them.

    python tests/golden/make_golden_letor.py /path/to/ptranking-checkout

For every file the unmodified reference ``iter_queries`` (ptranking/data/data_utils.py:420-549) runs on the CPU for each
config, and the npz keeps the file's bytes and, per config, the qids, offsets, X (float32) and y (float32) of the
result.  X is stored once per file and scaler, for the config that keeps every query unsorted: the other configs' rows are
those rows, of their kept queries (reordered within each query when presorted -- the reference's tie order is random,
np_arg_shuffle_ties), so they keep qids, offsets and labels only.  No test imports the reference: only this data is committed."""
import io
import os
import sys
import tempfile

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "letor.npz")
HALFWAY = ["9007199254740993", "2.2250738585072011e-308", "0.30000000000000001665", "1.00000000000000011102230246251565",
           "-4503599627370497.5", "7.2057594037927933e16", "1.7976931348623157e308", "5e-324", "-0.0", "+12.5E-3",
           "123456789012345678901", "0.1", "1e22", ".5", "3."]


def _val(rng, i, j):
    k = (i * 7 + j * 3) % 17
    if k == 0:
        return HALFWAY[(i + j) % len(HALFWAY)]
    if k == 1:
        return "%.17g" % rng.standard_normal()
    if k == 2:
        return "%.3e" % (rng.standard_normal() * 10.0 ** rng.integers(-5, 6))
    return "%g" % round(float(rng.standard_normal() * 10), 6)


def _queries(rng, nq, lo, hi):
    qs = []
    for q in range(nq):
        qs.append(int(rng.integers(lo, hi)))
    return qs


def mslr(rng):
    """136 features, no comments; qid:010 next to qid:10, a recurring qid, repeated fids on one line, hard tokens."""
    lines = []
    qids = ["10", "010", "7", "abc", "10"]            # "10" recurs after others: grouped with its first block
    for qi, qid in enumerate(qids):
        for d in range(int(rng.integers(2, 5))):
            toks = [str(int(rng.integers(0, 5))), "qid:" + qid]
            toks += ["%d:%s" % (j + 1, _val(rng, len(lines), j)) for j in range(136)]
            if d == 0:
                toks += ["5:%s" % _val(rng, len(lines), 200)]   # repeated fid: the last value wins
            lines.append(" ".join(toks))
    return ("\n".join(lines) + "\n").encode()


def mq2008(rng):
    """46 features, '#docid = ... inc = ... prob = ...' comments, CRLF line ends."""
    lines = []
    for qid in ["1001", "1002", "1001", "1003"]:
        for d in range(int(rng.integers(2, 7))):
            toks = [str(int(rng.integers(0, 3))), "qid:" + qid] + ["%d:%s" % (j + 1, "%.6f" % rng.random()) for j in range(46)]
            lines.append(" ".join(toks) + " #docid = GX%03d-%02d inc = 1 prob = %.6f" % (d, d, rng.random()))
    return ("\r\n".join(lines) + "\r\n").encode()


def yahoo(rng):
    """Zero-indexed and sparse: features missing from lines, width set by one rare high id; no trailing newline."""
    lines = []
    for qid in ["1", "2", "3", "2"]:
        for d in range(int(rng.integers(2, 6))):
            fids = sorted(rng.choice(40, int(rng.integers(3, 10)), replace=False))
            toks = [str(int(rng.integers(0, 5))), "qid:" + qid] + ["%d:%s" % (f, _val(rng, d, f)) for f in fids]
            lines.append(" ".join(toks))
    lines[3] += " 699:0.25"
    return "\n".join(lines).encode()


def istella(rng):
    """1.79769313486e+308 values (clipped at 1e6 before scaling)."""
    lines = []
    for qid in ["5", "6", "5"]:
        for d in range(int(rng.integers(3, 6))):
            vals = ["1.79769313486e+308" if rng.random() < 0.15 else "%g" % round(float(rng.random() * 1e4), 3) for _ in range(30)]
            lines.append(" ".join([str(int(rng.integers(0, 5))), "qid:" + qid] + ["%d:%s" % (j + 1, v) for j, v in enumerate(vals)]))
    return ("\n".join(lines) + "\n").encode()


def mq_list(rng):
    """MSLETOR_LIST: labels are rank positions, turned into n - r."""
    lines = []
    for qid in ["20", "21"]:
        n = int(rng.integers(4, 9))
        for r in rng.permutation(n):
            toks = [str(int(r)), "qid:" + qid] + ["%d:%s" % (j + 1, "%.6f" % rng.random()) for j in range(46)]
            lines.append(" ".join(toks) + " #docid = L%d" % r)
    return ("\n".join(lines) + "\n").encode()


FORMATS = {"mslr": ("MSLRWEB30K", mslr), "mq2008": ("MQ2008_Super", mq2008), "yahoo": ("Set1", yahoo),
           "istella": ("Istella_S", istella), "mqlist": ("MQ2008_List", mq_list)}
# (scaler_id or None, min_docs, min_rele, binary_rele, unknown_as_zero): every scaler with and without clipping
CONFIGS = [(s, md, mr, b, u) for s in (None, "StandardScaler", "MinMaxScaler")
           for (md, mr, b, u) in ((0, 0, False, False), (3, 1, True, False), (0, 2, False, True), (4, 0, True, True))]


def config_name(cfg, presort):
    s, md, mr, b, u = cfg
    return "%s_md%d_mr%d_b%d_u%d_p%d" % (s or "none", md, mr, int(b), int(u), int(presort))


def data_dict(data_id, cfg):
    from ptranking.data.data_utils import get_data_meta
    s, md, mr, b, u = cfg
    d = dict(data_id=data_id, min_docs=md, min_rele=mr, binary_rele=b, unknown_as_zero=u, scale_data=s is not None,
             scaler_id=s, scaler_level="QUERY" if s else None)
    d.update(get_data_meta(data_id=data_id))
    return d


def main(ref):
    sys.path.insert(0, ref)
    import contextlib
    from ptranking.data.data_utils import iter_queries
    rng = np.random.default_rng(20261018)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for fmt, (data_id, make) in FORMATS.items():
            raw = make(rng)
            out[f"{fmt}/file"] = np.frombuffer(raw, dtype=np.uint8)
            out[f"{fmt}/data_id"] = np.array(data_id)
            path = os.path.join(tmp, fmt + ".txt")
            open(path, "wb").write(raw)
            for cfg in CONFIGS:
                for presort in (False, True):
                    np.random.seed(0)
                    with contextlib.redirect_stdout(io.StringIO()):
                        qs = iter_queries(in_file=path, presort=presort, data_dict=data_dict(data_id, cfg),
                                          scale_data=cfg[0] is not None, scaler_id=cfg[0],
                                          perquery_file=os.path.join(tmp, "none.np"), buffer=False)
                    key = f"{fmt}/{config_name(cfg, presort)}"
                    if presort:              # same queries as the unsorted config; labels now in presort order
                        out[key + "/y"] = np.concatenate([q[2] for q in qs]).astype(np.float32) if qs else np.zeros(0, np.float32)
                        continue
                    lens = [q[1].shape[0] for q in qs]
                    out[key + "/qids"] = np.array([q[0] for q in qs], dtype=object).astype(str) if qs else np.array([], dtype=str)
                    out[key + "/offsets"] = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
                    if cfg[1:] != (0, 0, False, False):   # rows: those of the scaler's unclipped config
                        out[key + "/y"] = np.concatenate([q[2] for q in qs]).astype(np.float32) if qs else np.zeros(0, np.float32)
                        continue
                    W = qs[0][1].shape[1] if qs else 0
                    out[key + "/X"] = np.concatenate([q[1] for q in qs]).astype(np.float32) if qs else np.zeros((0, W), np.float32)
                    out[key + "/y"] = np.concatenate([q[2] for q in qs]).astype(np.float32) if qs else np.zeros(0, np.float32)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/path/to/ptranking")
