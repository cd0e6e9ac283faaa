"""Rerank mode of the diversification driver (mirror of RerankDIVDataset, ptranking/ltr_diversification/util/div_data.py
:130-192).

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
