"""The device DIVDataset's fixture (tests/golden/make_golden_divdata.py) as the reference's input dicts, and a float64
restatement of the greedy ideal alpha-DCG order (get_div_ideal_ranking) with the lowest-position tie rule.

Fixture layout (divdata.npz): ``table`` [D, F] float64, document i is ``d<i>``; per query i: ``pool_<i>`` its table rows
in permutation order, ``q_<i>`` [1, F] float64, ``subs_<i>`` the number of subtopic entries of each pool position (-1:
the document is absent from q_doc_subtopics), ``sids_<i>`` the entries, and what the unmodified reference built:
``ref_order_<i>`` (positions in the pool without repeats, in its order), ``ref_docs_<i>`` and ``ref_rele_<i>`` (its fp32 tensors)."""
import numpy as np

ALPHA = 0.5
MAX_SUBTOPIC_ID = 20


def num_queries(z):
    return int(z["num_queries"])


def covers(z, i):
    """Query i's subtopic entries per pool position: a list of int lists, None where the document is absent."""
    subs, sids = z[f"subs_{i}"], z[f"sids_{i}"]
    out, e = [], 0
    for c in subs:
        if c < 0:
            out.append(None)
            continue
        out.append([int(s) for s in sids[e:e + c]])
        e += c
    return out


def input_dicts(z, qids=None):
    """-> (list_as_file, dictQueryRepresentation, dictDocumentRepresentation, dictQueryPermutaion,
    dictQueryDocumentSubtopics) as the driver loads them (subtopic ids as strings, representations [1, F] float64)."""
    table = z["table"]
    doc_reprs = {f"d{r}": table[r:r + 1] for r in range(table.shape[0])}
    qids = list(range(num_queries(z))) if qids is None else list(qids)
    q_reprs, perms, q_docs = {}, {}, {}
    for i in qids:
        pool = [f"d{r}" for r in z[f"pool_{i}"]]
        q_reprs[str(i)] = z[f"q_{i}"]
        perms[str(i)] = dict(alphaDCG=float(i), permutation=pool)
        q_docs[str(i)] = {doc: [str(s) for s in c] for doc, c in zip(pool, covers(z, i)) if c is not None}
    return qids, q_reprs, doc_reprs, perms, q_docs


def pool_covers(perms, q_docs, qid):
    """Query ``qid``'s pool as the dataset sees it -- the permutation without repeated documents -- and each document's
    subtopic ids as ints (None: absent from q_doc_subtopics)."""
    pool = list(dict.fromkeys(perms[str(qid)]["permutation"]))
    subs = q_docs[str(qid)]
    return pool, [None if doc not in subs else [int(s) for s in subs[doc]] for doc in pool]


def replay(cover, alpha=ALPHA, order=None):
    """The greedy in float64 -> (order, picked gain per step, max remaining gain per step, how many remaining positions
    reach that max).  Gains sum (1 - alpha) ** np.float64(count) over each position's entries in their order, as the
    reference does.  ``order`` None: pick the max, lowest position first; else replay the given order."""
    n = len(cover)
    entries = [c or [] for c in cover]
    k = max((len(c) for c in entries), default=0)
    ids = np.zeros((n, max(k, 1)), dtype=np.int64)
    has = np.zeros((n, max(k, 1)), dtype=bool)
    for d, c in enumerate(entries):
        ids[d, :len(c)] = c
        has[d, :len(c)] = True
    pw = np.asarray([(1 - alpha) ** np.float64(c) for c in range(sum(map(len, entries)) + 1)])
    cnt = np.zeros(MAX_SUBTOPIC_ID + 1, dtype=np.int64)          # index by id, slot 0 unused
    placed = np.zeros(n, dtype=bool)
    out, picked, best, ties = [], [], [], []
    for step in range(n):
        g = np.zeros(n)
        for j in range(ids.shape[1]):                             # sequential over entries, as the reference sums
            g = np.where(has[:, j], g + pw[cnt[ids[:, j]]], g)
        g[placed] = -1.0
        mx = g.max()
        d = int(np.argmax(g)) if order is None else int(order[step])
        assert not placed[d], f"position {d} placed twice"
        out.append(d)
        picked.append(g[d])
        best.append(mx)
        ties.append(int(np.sum(g == mx)))
        placed[d] = True
        for s in entries[d]:
            cnt[s] += 1
    return np.asarray(out), np.asarray(picked), np.asarray(best), np.asarray(ties)


def tie_free(cover, order, alpha=ALPHA):
    """Whether the greedy meets no tie along ``order``: every step's max is reached by one remaining position."""
    _, _, _, ties = replay(cover, alpha, order)
    return bool(np.all(ties == 1))


def to_matrix(cover, order):
    """The reference's to_matrix of the pool in ``order``, float32: row s-1 = 1 where a document covers s, as many rows
    as the largest id present, 19 zero rows when no document has a subtopic."""
    m = max((s for c in cover if c for s in c), default=-1)
    R = np.zeros((MAX_SUBTOPIC_ID, len(order)), dtype=np.float32)
    for col, d in enumerate(order):
        for s in cover[d] or ():
            R[s - 1, col] = 1.0
    return R[0:m]
