"""The diversification driver's datasets on the device: DIVDataset (ptranking/ltr_diversification/util/div_data.py:53-127)
and rerank mode's RerankDIVDataset (:130-192).

DIVDataset
----------
The reference builds every split query by query in Python: the greedy ideal alpha-DCG order of each pool
(get_div_ideal_ranking, O(n^2 m) Python loops), a vstack of the document rows and the subtopic matrix (to_matrix),
then DiversityNeuralRanker._split copies them to the device.  This drop-in keeps the constructor.  The document table
is indexed and uploaded once per ``dictDocumentRepresentation`` object (shared by every split of every fold while a
dataset holds it); each split turns its permutations and ``q_doc_subtopics`` into int arrays on the host, then one
ptrb200_div_ideal_order launch orders every query and one ptrb200_div_pack_split launch writes the q rows, the doc rows
in ideal order and the relevance blocks, which _split adopts as they are.  The order is read back once per split for
``perm_docs``.

Differences from the reference, by design:
* ties between equal gains go to the lower position in the permutation as given; the reference takes the first in
  ``set`` iteration order, which depends on string hashing (PYTHONHASHSEED);
* subtopic ids outside 1..20 are refused (the reference raises beyond 20 and silently maps 0 to the 20th row);
* ``add_noise`` draws its Gaussian noise on the device from a counter-based stream keyed by ``noise_seed`` (drawn from
  torch's CPU generator when not given), so the same seed gives the same rows; the reference uses torch.normal;
* ``buffer`` is accepted and writes no pickle.

RerankDIVDataset
----------------
The reference's RerankDIVDataset runs the first-stage ranker (the "discriminator") on every ``__getitem__``: one
``div_predict`` for the query, a device-to-host copy of its scores, a CPU ``torch.sort`` and the first ``rerank_k``
indices re-sorted ascending.  This drop-in keeps its constructor and the underlying DIVDataset pool, but selects for a
whole split at once on the device: the pool is packed once (diversity_ranker._Split with its raw rows), the
discriminator scores all of it in one batched forward in its current mode (its own feature order and
``split_sort_keys``, so DivProbRanker's ExpRele / RERAR / RiskAware keys apply), one ptrb200_div_rerank_select launch
sequence picks every query's top ``rerank_k`` rows and one ptrb200_div_rerank_gather copies the selected rows and
relevance columns.  DiversityNeuralRanker._split asks for a new selection on every pass over the dataset (each training
epoch, each evaluation call), as the reference's per-access selection gives a new draw whenever the discriminator's
dropout is live.

Differences from the reference, by design:
* ties at the ``rerank_k`` boundary go to the lower row index (key descending, then index ascending); the reference's
  CPU ``torch.sort`` is not asked to be stable;
* a selection of one document keeps its axes: doc rows [1, F] and relevance [m, 1], where the reference's
  ``torch.squeeze`` of the index gives [F] and [m].
"""
from __future__ import annotations

import itertools
import weakref

import numpy as np
import torch
import torch.utils.data as data

from .. import ops
from .base.diversity_ranker import _Split


class _Selection:
    """One selection pass on the device: the kept rows ``docs`` [sum c_q, F] (host counts ``lens``, device
    ``sel_offsets`` / within-query indices ``sel_idx``), the relevance blocks ``rele`` ([m_q, c_q] each, host offsets
    ``rele_offsets_host``), their relevance mass ``rele_sum`` (host) and the first-stage ``keys`` they were selected by."""

    def __init__(self, keys, lens, sel_offsets, sel_idx, docs, rele, rele_offsets_host, rele_sum):
        self.keys, self.lens, self.sel_offsets, self.sel_idx = keys, lens, sel_offsets, sel_idx
        self.docs, self.rele, self.rele_offsets_host, self.rele_sum = docs, rele, rele_offsets_host, rele_sum
        self.offsets_host = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


class RerankDIVDataset(data.Dataset):
    """The reference's constructor (div_data.py:135-149): a DIVDataset pool built by the reference's own DIVDataset, the
    ``discriminator`` (a first-stage ranker of this package, on its device) and ``eval_dict['rerank_k']``.  ``gpu`` and
    ``device`` are kept as given; the pool lives on the discriminator's device."""

    def __init__(self, split_type=None, list_as_file=None, data_id=None, data_dict=None, fold_dir=None, presort=True,
                 alpha=0.5, dictQueryRepresentation=None, dictDocumentRepresentation=None, dictQueryPermutaion=None,
                 dictQueryDocumentSubtopics=None, buffer=True, discriminator=None, eval_dict=None, gpu=False,
                 device=None):
        from ptranking.ltr_diversification.util.div_data import DIVDataset   # the reference must be importable
        pool = DIVDataset(split_type=split_type, list_as_file=list_as_file, data_id=data_id, data_dict=data_dict,
                          fold_dir=fold_dir, presort=presort, alpha=alpha,
                          dictQueryRepresentation=dictQueryRepresentation,
                          dictDocumentRepresentation=dictDocumentRepresentation,
                          dictQueryPermutaion=dictQueryPermutaion,
                          dictQueryDocumentSubtopics=dictQueryDocumentSubtopics, buffer=buffer)
        self._init(pool.list_torch_Qs, discriminator, eval_dict['rerank_k'], presort, gpu, device)

    @classmethod
    def from_queries(cls, list_torch_Qs, discriminator, rerank_k, presort=True, gpu=False, device=None):
        """A rerank dataset over in-memory query tuples (qid, q_repr, perm_docs, doc_reprs, alphaDCG, q_doc_subtopics,
        q_doc_rele_mat), as a DIVDataset holds them in ``list_torch_Qs``."""
        ds = cls.__new__(cls)
        ds._init(list(list_torch_Qs), discriminator, rerank_k, presort, gpu, device)
        return ds

    def _init(self, list_torch_Qs, discriminator, rerank_k, presort, gpu, device):
        assert discriminator is not None
        if int(rerank_k) < 1:
            raise ValueError(f"rerank_k={rerank_k} must be >= 1")
        self.list_torch_Qs = list_torch_Qs
        self.presort = presort
        self.discriminator = discriminator
        self.rerank_k = int(rerank_k)
        self.gpu, self.device = gpu, device
        self._pools, self._selection = {}, None

    def __len__(self):
        return len(self.list_torch_Qs)

    def pool(self):
        """The packed pool in the discriminator's feature order, built once per order and device."""
        d = self.discriminator
        key = (str(d.device), bool(d.split_list_order()))
        if key not in self._pools:
            self._pools[key] = _Split(self.list_torch_Qs, d.device, key[1], keep_rows=True)
        return self._pools[key]

    def select(self):
        """One selection pass over the whole pool: one discriminator forward in its current mode, one select and one
        gather launch sequence.  The result becomes the current selection and is returned."""
        pool = self.pool()
        keys = self.discriminator.split_keys(pool)
        lens = np.minimum(pool.lens_host, self.rerank_k)
        sizes = pool.sub_counts_host * lens
        _, sel_offsets, sel_idx = ops.div_rerank_select(keys, pool.offsets, pool.max_len, self.rerank_k,
                                                        total=int(lens.sum()))
        docs, rele = ops.div_rerank_gather(pool.docs, pool.offsets, sel_offsets, sel_idx, pool.rele,
                                           rele_numel=int(sizes.sum()))
        rele_offsets_host = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        # relevance mass per query for the skip rules: one float64 prefix sum and one device-to-host copy per pass
        cs = torch.cumsum(rele.rele.double(), 0)
        cs = torch.cat([torch.zeros(1, dtype=torch.float64, device=cs.device), cs])
        ro = torch.from_numpy(rele_offsets_host).to(cs.device)
        rele_sum = (cs[ro[1:]] - cs[ro[:-1]]).cpu().numpy()
        self._selection = _Selection(keys, lens, sel_offsets, sel_idx, docs, rele, rele_offsets_host, rele_sum)
        return self._selection

    def rerank_split(self, device, list_order):
        """A new selection as the second-stage ranker's packed split (DiversityNeuralRanker._split)."""
        pool, sel = self.pool(), self.select()
        perm_docs = [None] * len(pool)                       # the reference hands the second stage no perm_docs
        rele = ops.SubtopicRele(sel.rele.rele.to(device), sel.rele.rele_offsets.to(device),
                                sel.rele.sub_counts.to(device), sel.rele.max_sub)
        return _Split.from_rows(pool.qids, perm_docs, pool.q.to(device), sel.docs.to(device), sel.lens, rele,
                                sel.rele_sum, list_order)

    def __getitem__(self, index):
        """The reference's 7-tuple over the current selection (made now if there is none): doc rows [c, F] and the
        relevance columns [m, c] are device views; perm_docs and q_doc_subtopics are None, as in the reference."""
        sel = self._selection if self._selection is not None else self.select()
        qid, q_repr, _, _, alphaDCG, _, _ = self.list_torch_Qs[index]
        o0, o1 = int(sel.offsets_host[index]), int(sel.offsets_host[index + 1])
        r0, r1 = int(sel.rele_offsets_host[index]), int(sel.rele_offsets_host[index + 1])
        rele = sel.rele.rele[r0:r1].view(int(self.pool().sub_counts_host[index]), o1 - o0)
        return qid, q_repr, None, sel.docs[o0:o1], alphaDCG, None, rele


# ---------------------------------------------------------------------------------------------------------------- #
# DIVDataset
# ---------------------------------------------------------------------------------------------------------------- #
TREC_DIV = ('WT_Div_0912_Implicit', 'WT_Div_0912_Explicit')   # the data ids the reference's DIVDataset accepts
MAX_SUBTOPIC_ID = 20                                         # the reference's np.zeros(20) cover counts
EMPTY_POOL_ROWS = MAX_SUBTOPIC_ID - 1                        # to_matrix without subtopics returns rele_mat[0:-1]


class _DocTable:
    """A ``dictDocumentRepresentation``: doc id -> row ``index`` (host) and the rows as one fp32 [D, F] device tensor,
    uploaded on first use per device (rounded once on the host, as the reference's FloatTensor rounds each row)."""

    def __init__(self, doc_reprs):
        self.source, self.size = doc_reprs, len(doc_reprs)
        self.index = {doc: i for i, doc in enumerate(doc_reprs)}
        self._rows = None
        self._device = {}

    def rows(self):
        if self._rows is None:
            rows = np.vstack([np.asarray(v, dtype=np.float64).reshape(1, -1) for v in self.source.values()])
            self._rows = rows.astype(np.float32)
        return self._rows

    def on(self, device):
        key = str(device)
        if key not in self._device:
            self._device[key] = torch.from_numpy(self.rows()).to(device)
        return self._device[key]


# dicts cannot be weakly referenced, so the cache holds the tables weakly instead: a table lives while a dataset uses
# it, and it keeps its dict alive meanwhile, so the id in its key cannot be reused under it
_doc_tables = weakref.WeakValueDictionary()


def doc_table(doc_reprs) -> _DocTable:
    """The cached table of ``doc_reprs`` (the same dict object, unchanged in size), else a new one."""
    t = _doc_tables.get(id(doc_reprs))
    if t is None or t.source is not doc_reprs or t.size != len(doc_reprs):
        t = _doc_tables[id(doc_reprs)] = _DocTable(doc_reprs)
    return t


_pw_cache = {}


def alpha_powers(alpha: float, length: int) -> np.ndarray:
    """(1 - alpha)^c for c < length as the reference computes each gain term: a Python float raised to a numpy float64
    cover count."""
    pw = _pw_cache.get(alpha)
    if pw is None or pw.size < length:
        pw = np.asarray([(1 - alpha) ** np.float64(c) for c in range(max(length, 64))], dtype=np.float64)
        _pw_cache[alpha] = pw
    return pw[:length]


class HostSplit:
    """A split's host arrays: pool positions of query q are offsets[q] .. offsets[q+1]-1, ``rows`` their table rows,
    ``sub_offsets`` / ``sub_ids`` their subtopic CSR (ids in 1..20), ``sub_counts`` the to_matrix row count m_q,
    ``rele_offsets`` the exclusive scan of m_q n_q, ``rele_sum`` the number of ones in each block, ``q_rows`` [B, F]
    fp32, and per query the qid, the pool (doc ids, duplicates dropped as the reference's set() drops them), alphaDCG
    and q_doc_subtopics."""

    def __init__(self, list_as_file, table, dictQueryRepresentation, dictQueryPermutaion, dictQueryDocumentSubtopics):
        self.qids, self.pools, self.alpha_dcgs, self.subtopics = [], [], [], []
        rows, counts, ids, lens, q_rows = [], [], [], [], []
        for qid in list_as_file:
            key = str(qid)
            pool = dictQueryPermutaion[key]['permutation']
            if len(set(pool)) != len(pool):
                pool = list(dict.fromkeys(pool))
            if not pool:
                raise ValueError(f"query {qid}: empty permutation")
            q_doc_subtopics = dictQueryDocumentSubtopics[key]
            try:
                rows.append(np.fromiter(map(table.index.__getitem__, pool), dtype=np.int32, count=len(pool)))
            except KeyError as e:
                raise ValueError(f"query {qid}: document {e.args[0]!r} is not in dictDocumentRepresentation") from None
            covers = [q_doc_subtopics.get(doc) or () for doc in pool]
            counts.append(np.fromiter(map(len, covers), dtype=np.int64, count=len(pool)))
            q_ids = np.fromiter(map(int, itertools.chain.from_iterable(covers)), dtype=np.int64)
            bad = q_ids[(q_ids < 1) | (q_ids > MAX_SUBTOPIC_ID)]
            if bad.size:
                raise ValueError(f"query {qid}: subtopic id {int(bad[0])} outside 1..{MAX_SUBTOPIC_ID}")
            ids.append(q_ids)
            lens.append(len(pool))
            q_rows.append(np.asarray(dictQueryRepresentation[key], dtype=np.float64).reshape(1, -1))
            self.qids.append(qid)
            self.pools.append(pool)
            self.alpha_dcgs.append(dictQueryPermutaion[key]['alphaDCG'])
            self.subtopics.append(q_doc_subtopics)
        if not lens:
            raise ValueError("a split needs at least one query")
        if max(lens) > ops._lib.MAX_LIST_LEN:
            raise ValueError(f"a pool of {max(lens)} documents exceeds PTRB200_MAX_LIST_LEN={ops._lib.MAX_LIST_LEN}")
        B = len(lens)
        self.lens = np.asarray(lens, dtype=np.int64)
        self.offsets = np.concatenate([[0], np.cumsum(self.lens)]).astype(np.int64)
        self.rows = np.concatenate(rows)
        counts = np.concatenate(counts)
        self.sub_offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        sub_ids = np.concatenate(ids)
        self.sub_ids = sub_ids.astype(np.int32)
        self.q_rows = np.vstack(q_rows).astype(np.float32)
        # per query: its subtopic entries, the largest id among them (to_matrix's row count) and its distinct
        # (document, subtopic) pairs (the ones in its block)
        entries = self.sub_offsets[self.offsets]
        nnz = np.diff(entries)
        self.max_nnz = int(nnz.max())
        entry_q = np.repeat(np.arange(B), nnz)
        m = np.zeros(B, dtype=np.int64)
        np.maximum.at(m, entry_q, sub_ids)
        m[m == 0] = EMPTY_POOL_ROWS
        self.sub_counts = m.astype(np.int32)
        pairs = np.unique(np.repeat(np.arange(self.offsets[-1]), counts) * 32 + sub_ids)
        self.rele_sum = np.bincount(np.searchsorted(self.offsets, pairs // 32, side='right') - 1,
                                    minlength=B).astype(np.float64)
        sizes = m * self.lens
        self.rele_numel = int(sizes.sum())
        self.rele_offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)

    def __len__(self):
        return len(self.qids)


class DIVDataset(data.Dataset):
    """The reference's constructor (div_data.py:58-60).  The split is built on ``device`` (default: the current CUDA
    device) when it is constructed; ``noise_seed`` keys ``add_noise``'s stream (default: drawn from torch's CPU
    generator, so torch.manual_seed fixes it)."""

    def __init__(self, split_type, list_as_file, data_id=None, data_dict=None, fold_dir=None, presort=True, alpha=0.5,
                 dictQueryRepresentation=None, dictDocumentRepresentation=None, dictQueryPermutaion=None,
                 dictQueryDocumentSubtopics=None, buffer=True, add_noise=False, std_delta=1.0, noise_seed=None,
                 device=None):
        if presort is not True:
            raise AssertionError("DIVDataset needs presort=True: it orders every pool by its ideal diversified ranking")
        if data_dict['data_id'] not in TREC_DIV:
            raise NotImplementedError(data_dict['data_id'])
        std = float(std_delta) if add_noise else 0.0
        if not (np.isfinite(std) and std >= 0.0):
            raise ValueError(f"std_delta={std_delta} must be finite and >= 0")
        self.presort, self.add_noise, self.split_type = presort, add_noise, split_type
        self.data_id = data_dict['data_id']
        table = doc_table(dictDocumentRepresentation)
        host = HostSplit(list_as_file, table, dictQueryRepresentation, dictQueryPermutaion, dictQueryDocumentSubtopics)
        if add_noise and noise_seed is None:
            noise_seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        self.noise_seed = noise_seed
        self._table, self._host = table, host
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self._build(float(alpha), std)

    def _build(self, alpha, std):
        h, dev = self._host, self.device
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
        offsets = up(h.offsets.astype(np.int32))
        sub_offsets = up(h.sub_offsets.astype(np.int32))
        sub_ids = up(np.concatenate([h.sub_ids, np.zeros(1, np.int32)]))   # never a null pointer
        sub_counts, rele_offsets = up(h.sub_counts), up(h.rele_offsets)
        order = ops.div_ideal_order(offsets, sub_offsets, sub_ids, up(alpha_powers(alpha, h.max_nnz + 1)),
                                    int(h.lens.max()))
        self.q, self.docs, self.rele = ops.div_pack_split(
            self._table.on(dev), up(h.q_rows), offsets, up(h.rows), order, sub_offsets, sub_ids, rele_offsets,
            sub_counts, h.rele_numel, int(h.sub_counts.max()), std_delta=std, seed=self.noise_seed or 0)
        self.order = order.cpu().numpy()
        self.perm_docs = [[h.pools[q][i] for i in self.order[h.offsets[q]:h.offsets[q + 1]]] for q in range(len(h))]

    def __len__(self):
        return len(self._host)

    def __getitem__(self, index):
        """The reference's 7-tuple (qid, q_repr [1, F], perm_docs, doc_reprs [n, F], alphaDCG, q_doc_subtopics,
        q_doc_rele_mat [m, n]) with device views for the tensors and perm_docs in the computed order."""
        h = self._host
        o0, o1 = int(h.offsets[index]), int(h.offsets[index + 1])
        r0, m = int(h.rele_offsets[index]), int(h.sub_counts[index])
        rele = self.rele.rele[r0:r0 + m * (o1 - o0)].view(m, o1 - o0)
        return (h.qids[index], self.q[index:index + 1], self.perm_docs[index], self.docs[o0:o1], h.alpha_dcgs[index],
                h.subtopics[index], rele)

    def device_split(self, device, list_order):
        """The packed split for DiversityNeuralRanker._split, from the rows built here (copied only when ``device``
        differs)."""
        h = self._host
        rele = self.rele
        if torch.device(device) != self.device:
            rele = ops.SubtopicRele(rele.rele.to(device), rele.rele_offsets.to(device), rele.sub_counts.to(device),
                                    rele.max_sub)
        return _Split.from_rows(h.qids, self.perm_docs, self.q.to(device), self.docs.to(device), h.lens, rele,
                                h.rele_sum, list_order)
