"""Length-bucketed batching: the input side of the hot path (SURVEY.md 8f-2).

The reference batches whole queries and asks every batch to hold lists of ONE length: ``LETORSampler`` draws
``batch_size`` queries of equal ``num_docs`` (ptranking/data/data_utils.py:683-742), and with the default settings a
query of 100+ documents travels alone (B = 1), which leaves a GPU launch-bound.  ``LengthBucketedBatches`` keeps the
contract the kernels rely on -- uniform n per batch, labels presorted descending per query (data_utils.py:205-232) --
but sizes B per bucket so that every batch carries about ``docs_per_batch`` documents (2^18 fills one H100; one step of
the default scorer then runs at its large-batch rate).  Batches are assembled once into pinned host memory, so
``NeuralRanker.train`` can stream them with asynchronous copies.  Host-side only: no device work happens here.
"""
from __future__ import annotations

from collections import defaultdict
from typing import Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

Query = Tuple[str, np.ndarray, np.ndarray]        # (qid, features [n, F], labels [n])


def presort_query(features: np.ndarray, labels: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """Order one query's documents by label, descending and stable -- the ``presort=True`` contract
    (data_utils.py:221-232) every loss kernel assumes."""
    order = np.argsort(-labels, kind="stable")
    return features[order], labels[order]


def _check_feature_dtype(dtype: torch.dtype) -> torch.dtype:
    if dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"feature_dtype must be torch.float32 or torch.bfloat16, got {dtype}")
    return dtype


def features_to(X: np.ndarray, dtype: torch.dtype):
    """One query's fp32 features as the loaders keep them: the numpy array itself for torch.float32; for torch.bfloat16 a
    bf16 tensor, converted once here (round to nearest even).  bf16 batches halve the pinned host memory and the
    host-to-device copy, and the scorer's layer-0 kernels read them natively, with the results the same values give in
    fp32.  Pass features that are already scaled: raw LETOR features lose precision in bf16."""
    return X if dtype == torch.float32 else torch.from_numpy(X).to(dtype)


def _as_tensor(Xq) -> torch.Tensor:
    return Xq if isinstance(Xq, torch.Tensor) else torch.from_numpy(Xq)


class LengthBucketedBatches:
    """Iterable of ``(qids, X[B,n,F], y[B,n])`` CPU batches (pinned when CUDA is available).

    queries         : iterable of (qid, features [n,F] float32, labels [n])
    docs_per_batch  : target B*n per batch; B = max(1, docs_per_batch // n), capped by ``max_queries``
    presort         : sort each query's documents by label first (set False when the data already is)
    shuffle_seed    : None keeps dataset order inside each bucket; an int reshuffles buckets and batch order per epoch
    drop_ragged     : drop the last, smaller batch of each length instead of emitting it
    rank / world    : data-parallel sharding -- every rank walks the same batch list and keeps batches rank::world,
                      so all ranks see the same number of batches per epoch (the last ``len % world`` are dropped)
    feature_dtype   : torch.float32 (default) or torch.bfloat16 -- see :func:`features_to`
    """

    def __init__(self, queries: Iterable[Query], docs_per_batch: int = 1 << 18, max_queries: Optional[int] = None,
                 presort: bool = True, shuffle_seed: Optional[int] = None, drop_ragged: bool = False,
                 rank: int = 0, world: int = 1, pin_memory: Optional[bool] = None,
                 feature_dtype: torch.dtype = torch.float32):
        if docs_per_batch < 1 or world < 1 or not (0 <= rank < world):
            raise ValueError("docs_per_batch >= 1 and 0 <= rank < world are required")
        self.feature_dtype = _check_feature_dtype(feature_dtype)
        self.docs_per_batch, self.max_queries = int(docs_per_batch), max_queries
        self.shuffle_seed, self.drop_ragged, self.rank, self.world = shuffle_seed, drop_ragged, rank, world
        self.pin = torch.cuda.is_available() if pin_memory is None else bool(pin_memory)
        self.epoch = 0
        self.buckets = defaultdict(list)                 # n -> [(qid, X, y)]
        self.num_features = None
        for qid, X, y in queries:
            X = np.ascontiguousarray(X, dtype=np.float32)
            y = np.ascontiguousarray(y, dtype=np.float32)
            if X.ndim != 2 or y.shape != (X.shape[0],):
                raise ValueError(f"query {qid}: features {X.shape} / labels {y.shape} do not describe one list")
            if X.shape[0] == 0:
                continue                                 # the reference skips empty queries as well (data_utils.py:150-155)
            if self.num_features is None:
                self.num_features = X.shape[1]
            elif X.shape[1] != self.num_features:
                raise ValueError(f"query {qid}: {X.shape[1]} features, expected {self.num_features}")
            if presort:
                X, y = presort_query(X, y)
            self.buckets[X.shape[0]].append((str(qid), features_to(X, self.feature_dtype), y))

    @classmethod
    def from_split(cls, split, docs_per_batch: int = 1 << 18, max_queries: Optional[int] = None,
                   shuffle_seed: Optional[int] = None, drop_ragged: bool = False, rank: int = 0, world: int = 1):
        """The same batches as the constructor given ``split``'s queries in order, built on the device from a
        :class:`ptranking_b200.letor.LetorSplit` with no host copy of the features.  The split is taken as read: presort
        it with ``read_letor(presort=True)``; the feature dtype is the split's."""
        self = cls([], docs_per_batch=docs_per_batch, max_queries=max_queries, presort=False, shuffle_seed=shuffle_seed,
                   drop_ragged=drop_ragged, rank=rank, world=world, pin_memory=False,
                   feature_dtype=split.X.dtype)
        self.device = split.X.device
        self.num_features = split.num_features
        for b in range(len(split)):
            qid, X, y = split.query(b)
            self.buckets[X.shape[0]].append((qid, X, y))
        return self

    def batch_size(self, n: int) -> int:
        B = max(1, self.docs_per_batch // n)
        return min(B, self.max_queries) if self.max_queries else B

    def _plan(self) -> List[Tuple[int, List[int]]]:
        rng = np.random.default_rng(self.shuffle_seed + self.epoch) if self.shuffle_seed is not None else None
        plan = []
        for n in sorted(self.buckets):
            idx = np.arange(len(self.buckets[n]))
            if rng is not None:
                rng.shuffle(idx)
            B = self.batch_size(n)
            for s in range(0, len(idx), B):
                chunk = idx[s: s + B]
                if len(chunk) < B and self.drop_ragged:
                    continue
                plan.append((n, chunk.tolist()))
        if rng is not None:
            rng.shuffle(plan)
        usable = len(plan) - len(plan) % self.world
        return plan[:usable][self.rank:: self.world]

    def __len__(self) -> int:
        return len(self._plan())

    def __iter__(self) -> Iterator[Tuple[List[str], torch.Tensor, torch.Tensor]]:
        plan = self._plan()
        self.epoch += 1
        for n, members in plan:
            qs = [self.buckets[n][i] for i in members]
            if getattr(self, "device", None) is not None:        # from_split: the queries are device views
                yield [q[0] for q in qs], torch.stack([q[1] for q in qs]), torch.stack([q[2] for q in qs])
                continue
            X = torch.empty((len(qs), n, self.num_features), dtype=self.feature_dtype, pin_memory=self.pin)
            y = torch.empty((len(qs), n), dtype=torch.float32, pin_memory=self.pin)
            for b, (_, Xq, yq) in enumerate(qs):
                X[b] = _as_tensor(Xq)
                y[b] = torch.from_numpy(yq)
            yield [q[0] for q in qs], X, y

    def stats(self) -> dict:
        """Fill statistics: queries, documents, batches, and the share of batches that reach the document target."""
        plan = self._plan() if self.world == 1 else None
        nq = sum(len(v) for v in self.buckets.values())
        nd = sum(n * len(v) for n, v in self.buckets.items())
        out = dict(queries=nq, docs=nd, lengths=len(self.buckets))
        if plan is not None:
            docs = [n * len(m) for n, m in plan]
            out.update(batches=len(plan), mean_docs_per_batch=float(np.mean(docs)) if docs else 0.0,
                       full_batches=float(np.mean([d >= 0.5 * self.docs_per_batch for d in docs])) if docs else 0.0)
        return out


def length_buckets(lens_desc: Sequence[int], edges: Sequence[int] = (128, 512)) -> List[Tuple[int, int, int]]:
    """[(q_begin, q_end, max_len)] over queries sorted by length DESCENDING: one bucket per length class
    (.., 128], (128, 512], (512, inf) -- the classes at which the pairwise-loss kernels change CTA size and schedule --
    classes holding fewer than 8 queries merged into their longer neighbour."""
    lens = np.asarray(lens_desc)
    if len(lens) == 0:
        return []
    cls = np.searchsorted(np.asarray(edges), lens, side="left")          # class index grows with length
    out: List[Tuple[int, int, int]] = []
    start = 0
    for i in range(1, len(lens) + 1):
        if i == len(lens) or cls[i] != cls[start]:
            if out and (out[-1][1] - out[-1][0] < 8):                    # the previous class is too small for a launch of its own
                b0, _, ml = out.pop()
                out.append((b0, i, ml))
            else:
                out.append((start, i, int(lens[start])))
            start = i
    return out


class RaggedBatches:
    """Iterable of ragged batches ``(qids, X[total,F], y[total], offsets[B+1] int32, max_len, buckets)`` -- variable-length
    lists inside ONE launch (SURVEY 8f-2).  Inside a batch the queries are ordered by length, longest first, and
    ``buckets`` = [(q_begin, q_end, max_len), ...] cuts that order into length classes, so the O(n^2) loss kernels can
    size their CTAs and pair schedule for each class instead of for the longest list of the batch (one launch per class,
    the long-list class on a side stream).

    The reference batches only queries of identical length (data_utils.py:683-742); on real collections (MSLR-WEB30K:
    1..1251 documents per query, mean 119.6, testing/data/testing_data_utils.py:318-326) equal-length buckets hold a
    handful of queries each and cannot fill a GPU.  Here queries are packed in dataset (or shuffled) order until about
    ``docs_per_batch`` documents are reached, whatever their lengths; the kernels address each query through the prefix
    offsets.  Same presort contract as :class:`LengthBucketedBatches`; rank-disjoint shards with equal batch counts.
    """

    def __init__(self, queries: Iterable[Query], docs_per_batch: int = 1 << 18, max_queries: Optional[int] = None,
                 presort: bool = True, shuffle_seed: Optional[int] = None, rank: int = 0, world: int = 1,
                 pin_memory: Optional[bool] = None, max_list_len: int = 4096, bucket_edges: Sequence[int] = (128, 512),
                 feature_dtype: torch.dtype = torch.float32):
        """``bucket_edges``: upper ends of the length classes a batch is cut into (:func:`length_buckets`).  The default
        suits the pairwise-loss kernels; the list scorer pads every class to its longest list and attention work grows
        with the square of that length, so it is better served by finer classes, e.g. (32, 64, 128, 256).
        ``feature_dtype``: torch.float32 (default) or torch.bfloat16 -- see :func:`features_to`."""
        if docs_per_batch < 1 or world < 1 or not (0 <= rank < world):
            raise ValueError("docs_per_batch >= 1 and 0 <= rank < world are required")
        self.feature_dtype = _check_feature_dtype(feature_dtype)
        if list(bucket_edges) != sorted(set(int(e) for e in bucket_edges)) or any(int(e) < 1 for e in bucket_edges):
            raise ValueError("bucket_edges must be increasing positive lengths")
        self.bucket_edges = tuple(int(e) for e in bucket_edges)
        self.docs_per_batch, self.max_queries = int(docs_per_batch), max_queries
        self.shuffle_seed, self.rank, self.world = shuffle_seed, rank, world
        self.pin = torch.cuda.is_available() if pin_memory is None else bool(pin_memory)
        self.epoch = 0
        self.queries: List[Tuple[str, np.ndarray, np.ndarray]] = []
        self.num_features = None
        for qid, X, y in queries:
            X = np.ascontiguousarray(X, dtype=np.float32)
            y = np.ascontiguousarray(y, dtype=np.float32)
            if X.ndim != 2 or y.shape != (X.shape[0],):
                raise ValueError(f"query {qid}: features {X.shape} / labels {y.shape} do not describe one list")
            if X.shape[0] == 0:
                continue
            if X.shape[0] > max_list_len:
                raise ValueError(f"query {qid}: {X.shape[0]} documents exceed the per-list kernel limit {max_list_len}")
            if self.num_features is None:
                self.num_features = X.shape[1]
            elif X.shape[1] != self.num_features:
                raise ValueError(f"query {qid}: {X.shape[1]} features, expected {self.num_features}")
            if presort:
                X, y = presort_query(X, y)
            self.queries.append((str(qid), features_to(X, self.feature_dtype), y))

    @classmethod
    def from_split(cls, split, docs_per_batch: int = 1 << 18, max_queries: Optional[int] = None,
                   shuffle_seed: Optional[int] = None, rank: int = 0, world: int = 1, max_list_len: int = 4096,
                   bucket_edges: Sequence[int] = (128, 512)):
        """The same batches as the constructor given ``split``'s queries in order, built on the device from a
        :class:`ptranking_b200.letor.LetorSplit` with no host copy of the features.  The split is taken as read: presort
        it with ``read_letor(presort=True)``; the feature dtype is the split's."""
        self = cls([], docs_per_batch=docs_per_batch, max_queries=max_queries, presort=False, shuffle_seed=shuffle_seed,
                   rank=rank, world=world, pin_memory=False, max_list_len=max_list_len, bucket_edges=bucket_edges,
                   feature_dtype=split.X.dtype)
        if split.max_len > max_list_len:
            raise ValueError(f"a query of {split.max_len} documents exceeds the per-list kernel limit {max_list_len}")
        self.device = split.X.device
        self.num_features = split.num_features
        self.queries = [split.query(b) for b in range(len(split))]
        return self

    def _plan(self) -> List[List[int]]:
        idx = np.arange(len(self.queries))
        if self.shuffle_seed is not None:
            np.random.default_rng(self.shuffle_seed + self.epoch).shuffle(idx)
        plan, cur, docs = [], [], 0
        for i in idx:
            n = self.queries[i][1].shape[0]
            if cur and (docs + n > self.docs_per_batch or (self.max_queries and len(cur) >= self.max_queries)):
                plan.append(cur)
                cur, docs = [], 0
            cur.append(int(i))
            docs += n
        if cur:
            plan.append(cur)
        usable = len(plan) - len(plan) % self.world
        return plan[:usable][self.rank:: self.world]

    def __len__(self) -> int:
        return len(self._plan())

    def __iter__(self):
        plan = self._plan()
        self.epoch += 1
        for members in plan:
            qs = sorted((self.queries[i] for i in members), key=lambda q: -q[1].shape[0])
            lens = np.array([q[1].shape[0] for q in qs], dtype=np.int64)
            total = int(lens.sum())
            if getattr(self, "device", None) is not None:        # from_split: the queries are device views
                offsets = torch.zeros(len(qs) + 1, dtype=torch.int32)
                offsets[1:] = torch.from_numpy(np.cumsum(lens)).to(torch.int32)
                yield ([q[0] for q in qs], torch.cat([q[1] for q in qs]), torch.cat([q[2] for q in qs]),
                       offsets.to(self.device), int(lens.max()), length_buckets(lens, edges=self.bucket_edges))
                continue
            X = torch.empty((total, self.num_features), dtype=self.feature_dtype, pin_memory=self.pin)
            y = torch.empty((total,), dtype=torch.float32, pin_memory=self.pin)
            offsets = torch.zeros(len(qs) + 1, dtype=torch.int32, pin_memory=self.pin)
            offsets[1:] = torch.from_numpy(np.cumsum(lens)).to(torch.int32)
            o = 0
            for _, Xq, yq in qs:
                X[o: o + Xq.shape[0]] = _as_tensor(Xq)
                y[o: o + Xq.shape[0]] = torch.from_numpy(yq)
                o += Xq.shape[0]
            yield [q[0] for q in qs], X, y, offsets, int(lens.max()), length_buckets(lens, edges=self.bucket_edges)

    def stats(self) -> dict:
        lens = np.array([q[1].shape[0] for q in self.queries])
        out = dict(queries=len(lens), docs=int(lens.sum()), min_len=int(lens.min()) if len(lens) else 0,
                   max_len=int(lens.max()) if len(lens) else 0, mean_len=float(lens.mean()) if len(lens) else 0.0)
        if self.world == 1:
            plan = self._plan()
            docs = [int(sum(self.queries[i][1].shape[0] for i in m)) for m in plan]
            out.update(batches=len(plan), mean_docs_per_batch=float(np.mean(docs)) if docs else 0.0)
        return out
