"""DiversityNeuralRanker with the pointwise or the list scorer (mirror of
ptranking/ltr_diversification/base/diversity_ranker.py, div_point_ranker.py, div_list_ranker.py and the
diversified-ranking methods of base/ranker.py:265-475, :655-700).

The reference walks a DIVDataset query by query: one scorer forward per query, and for evaluation a device-to-host copy
and a CPU metric per query.  Here a split is packed once into device tensors -- the [q, q*d, d] scorer input of every
document (ops.div_features), ragged offsets and the subtopic relevance blocks -- and cached per dataset object.
Evaluation is one scorer forward and one metric launch per split; training keeps the reference's one step per query by
default.  The reference's BN normalises each query over its own documents because it scores one query per call; the
scorer's per-query BN mode (StackedFFNet ``bn_per_query``) keeps that when many queries share a launch.  The list
scorer (sf_id='listsf', div_list_ranker.py) reads the list-order rows [q, d, q*d] instead, which are then the only
features a listsf ranker builds for a split.
"""
from __future__ import annotations

import os
import weakref

import numpy as np
import torch

from ... import ops
from ...base.point_ranker import PointNeuralRanker
from ...base.utils import StackedFFNet
from .div_list_ranker import ATTN_BUDGET_BYTES, DivListNeuralRanker, check_listsf_config


class _Split:
    """One DIVDataset on the device: X [total, 3F] scorer input ([q, q*d, d]; [q, d, q*d] with ``list_order``, the
    list scorer's encoder input), int32 offsets [Q+1] (device) and their host copy, the subtopic relevance blocks, host
    qids / perm_docs and the per-query relevance mass (host, for the skip rules)."""

    def __init__(self, data, device, list_order=False, keep_rows=False):
        """``keep_rows``: also keep the raw rows ``q`` [Q, F] and ``docs`` [total, F] on the device (a rerank pool)."""
        qids, perm_docs, q_reprs, docs, mats = [], [], [], [], []
        for qid, q_repr, q_perm_docs, doc_reprs, _alpha_dcg, _subtopics, q_doc_rele_mat in data:
            qids.append(qid)
            perm_docs.append(q_perm_docs)
            q_reprs.append(torch.as_tensor(q_repr, dtype=torch.float32).reshape(1, -1))
            docs.append(torch.as_tensor(doc_reprs, dtype=torch.float32))
            mats.append(torch.as_tensor(q_doc_rele_mat, dtype=torch.float32))
        lens = [int(d.shape[0]) for d in docs]
        rele_sum = np.asarray([float(torch.sum(r)) for r in mats])      # reference's torch.sum, fp32
        self.sub_counts_host = np.asarray([int(r.shape[0]) for r in mats], dtype=np.int64)
        q = torch.cat(q_reprs).to(device) if q_reprs else torch.zeros(0, 1, device=device)
        d = torch.cat(docs).to(device) if docs else torch.zeros(0, 1, device=device)
        self._setup(qids, perm_docs, q, d, lens, ops.SubtopicRele.pack(mats, device), rele_sum, list_order)
        if keep_rows:
            self.q, self.docs = q, d

    @classmethod
    def from_rows(cls, qids, perm_docs, q, docs, lens, rele, rele_sum, list_order=False):
        """A split from device rows: q [Q, F], docs [total, F] cut by the host list lengths ``lens``, the relevance
        blocks ``rele`` (ops.SubtopicRele) and their host relevance mass ``rele_sum`` (a rerank selection)."""
        sp = cls.__new__(cls)
        sp._setup(list(qids), list(perm_docs), q, docs, lens, rele, np.asarray(rele_sum, dtype=np.float64), list_order)
        return sp

    def _setup(self, qids, perm_docs, q, d, lens, rele, rele_sum, list_order):
        device = d.device
        self.qids, self.perm_docs = qids, perm_docs
        lens = [int(n) for n in lens]
        self.offsets_host = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        self.lens_host = np.asarray(lens, dtype=np.int64)
        self.max_len = max(lens, default=1)
        self.rele_sum = rele_sum
        self.offsets = torch.from_numpy(self.offsets_host.astype(np.int32)).to(device)
        self.lens = torch.from_numpy(self.lens_host.astype(np.int32)).to(device)
        self.rele = rele
        build = ops.div_list_features if list_order else ops.div_features
        self.X = build(q, d, offsets=self.offsets, max_len=self.max_len)
        self._steps, self._plans = {}, {}

    def __len__(self):
        return len(self.qids)

    def steps(self, queries_per_step):
        """Training batches: runs of at most ``queries_per_step`` consecutive queries with sum(R) >= 1 (a batch never
        spans a skipped query), as (q0, q1, row0, row1, device offsets rebased to row0, longest list)."""
        if queries_per_step not in self._steps:
            out, run = [], []
            for q in range(len(self)):
                if self.rele_sum[q] < 1.0:
                    if run:
                        out.append(run)
                    run = []
                    continue
                run.append(q)
                if len(run) == queries_per_step:
                    out.append(run)
                    run = []
            if run:
                out.append(run)
            steps = []
            for r in out:
                q0, q1 = r[0], r[-1] + 1
                o = self.offsets_host[q0:q1 + 1]
                off = torch.from_numpy((o - o[0]).astype(np.int32)).to(self.offsets.device)
                steps.append((q0, q1, int(o[0]), int(o[-1]), off, int(self.lens_host[q0:q1].max())))
            self._steps[queries_per_step] = steps
        return self._steps[queries_per_step]

    def plan(self, q0, q1, ranker):
        """The list scorer's layout of queries [q0, q1) (div_list_ranker.ListPlan), built once per budget."""
        key = (q0, q1, ranker.attn_budget_bytes)
        if key not in self._plans:
            self._plans[key] = ranker.list_plan(self.offsets_host[q0:q1 + 1])
        return self._plans[key]


class DiversityNeuralRanker(PointNeuralRanker, DivListNeuralRanker):
    """sf_id 'pointsf' (stacked FF net over [q, q*d, d]) or 'listsf' (MHSA encoder over [q, d, q*d], then a univariate
    FF net over [q, d, q*d, enc]; DivListNeuralRanker)."""

    def __init__(self, id='DiversityNeuralRanker', sf_para_dict=None, weight_decay=1e-3, gpu=False, device=None):
        self.sf_id = sf_para_dict['sf_id']
        assert self.sf_id in ['pointsf', 'listsf']
        if 'listsf' == self.sf_id:
            check_listsf_config(sf_para_dict['listsf'])
        super().__init__(id=id, sf_para_dict=sf_para_dict, weight_decay=weight_decay, gpu=gpu, device=device)
        if 'pointsf' == self.sf_id:
            # the scorer reads the concatenation [q, q*d, d] (diversity_ranker.py:22-23)
            self.sf_para_dict[self.sf_id]['num_features'] *= 3
        else:
            # the list scorer widens its own layers (div_list_ranker.py:26); num_features stays F (diversity_ranker.py:24-25)
            self.encoder_type = self.sf_para_dict['listsf']['encoder_type']
        self.queries_per_step = 1
        self.attn_budget_bytes = ATTN_BUDGET_BYTES
        self._splits, self._weak_splits = {}, weakref.WeakKeyDictionary()

    def init(self):
        if 'pointsf' == self.sf_id:
            return PointNeuralRanker.init(self)
        self.list_sf = self.ini_listsf(**self.sf_para_dict['listsf'])
        self.config_optimizer()

    def get_parameters(self):
        if 'pointsf' == self.sf_id:
            return PointNeuralRanker.get_parameters(self)
        return self.list_parameters()

    # ---- scorer ------------------------------------------------------------------------------------------------- #
    def ini_pointsf(self, num_features=None, h_dim=100, out_dim=1, num_layers=3, AF='R', TL_AF='S', apply_tl_af=False,
                    BN=True, bn_type=None, bn_affine=False, dropout=0.1):
        """point_ranker.py:30-42, with BN statistics per query (the reference scores one query per call)."""
        ff_dims = [num_features] + [h_dim] * num_layers + [out_dim]
        return StackedFFNet(ff_dims, AF=AF, TL_AF=TL_AF, apply_tl_af=apply_tl_af, dropout=dropout, BN=BN,
                            bn_type=bn_type, bn_affine=bn_affine, device=self.device,
                            bn_per_query=bool(BN) and bn_type == 'BN', pad_output=True)

    def div_forward(self, q_repr, doc_reprs):
        """div_point_ranker.py:14-24 / div_list_ranker.py:61-85: q_repr [1,F], doc_reprs [n,F] -> [1,n]."""
        if 'listsf' == self.sf_id:
            return self.list_div_forward(q_repr, doc_reprs)
        num_docs = doc_reprs.size(0)
        X = ops.div_features(q_repr.reshape(1, -1), doc_reprs.unsqueeze(0))
        return self.point_sf(X).view(-1, num_docs)

    def div_predict(self, q_repr, doc_reprs):
        """ranker.py:690-695."""
        return self.div_forward(q_repr, doc_reprs)

    def div_forward_ragged(self, X, offsets, max_len):
        """[total, 3F] scorer input of a ragged batch -> flat scores [total] (per-query BN statistics)."""
        return self.point_sf(X, offsets=offsets, max_len=max_len).view(-1)

    def split_list_order(self):
        """Whether a split's scorer input is packed as [q, d, q*d] (True) or [q, q*d, d]: the list scorer reads the
        former, the pointwise scorer of DiversityNeuralRanker the latter.  A subclass whose pointwise scorer reads the
        list order overrides this."""
        return 'listsf' == self.sf_id

    def split_sort_keys(self, preds, sp):
        """The sort keys of a packed split from its scorer output ``preds`` (flat, as div_forward_ragged / list_scores
        return it), in the split's row order.  The scores themselves by default."""
        return preds

    def split_keys(self, sp):
        """The sort keys of every row of a packed split from one scorer forward in the ranker's current mode (flat, in
        the split's row order)."""
        with torch.no_grad():
            if 'listsf' == self.sf_id:
                preds = self.list_scores(sp.X, sp.plan(0, len(sp), self))
            else:
                preds = self.div_forward_ragged(sp.X, sp.offsets, sp.max_len)
            return self.split_sort_keys(preds, sp)

    def _split(self, data):
        """The packed device copy of ``data``, built on first use and cached for the dataset object (weakly where the
        object allows it, so the device copies of a finished fold's splits go with their datasets).  A rerank dataset
        (div_data.RerankDIVDataset) selects its pools anew on every call: one pass over the data.  A device-built
        dataset (div_data.DIVDataset) hands over its packed rows as they are."""
        rerank = getattr(data, 'rerank_split', None)
        if rerank is not None:
            return rerank(self.device, self.split_list_order())
        try:
            sp = self._weak_splits.get(data)
            if sp is None:
                device_split = getattr(data, 'device_split', None)
                sp = self._weak_splits[data] = (_Split(data, self.device, self.split_list_order())
                                                if device_split is None
                                                else device_split(self.device, self.split_list_order()))
            return sp
        except TypeError:                           # e.g. a plain list of query tuples
            hit = self._splits.get(id(data))
            if hit is None or hit[0] is not data:
                hit = self._splits[id(data)] = (data, _Split(data, self.device, self.split_list_order()))
            return hit[1]

    # ---- training ----------------------------------------------------------------------------------------------- #
    def div_train(self, train_data, epoch_k=None, queries_per_step=None):
        """ranker.py:632-657: one epoch.  Queries with sum(R) < 1 are skipped, the epoch loss is the sum of the step
        losses over len(train_data), and on every stop_check_freq-th epoch the scores of each step are checked, the
        epoch ending at the first failing one.  ``queries_per_step`` (default: the ranker's ``queries_per_step``,
        1 = the reference) > 1 trains consecutive queries as one ragged batch: one scorer call with per-query BN
        statistics, one loss launch and one optimizer step on the sum of their losses.  The step losses are read back
        once per epoch (the reference reads each with .item()).  The list scorer runs the step's queries through the
        encoder padded per length class, then uni_sf over their flat rows."""
        self.train_mode()
        qps = int(queries_per_step or self.queries_per_step)
        if qps < 1:
            raise ValueError("queries_per_step must be >= 1")
        sp = self._split(train_data)
        check = epoch_k is not None and epoch_k % self.stop_check_freq == 0
        losses, stop_training = [], False
        for q0, q1, r0, r1, off, max_len in sp.steps(qps):
            X = sp.X[r0:r1]
            if 'listsf' == self.sf_id:
                batch_pred = self.list_scores(X, sp.plan(q0, q1, self))
                if q1 - q0 == 1:
                    batch_pred, layout = batch_pred.view(1, -1), {}
                else:
                    layout = dict(offsets=off, max_len=max_len)
            elif q1 - q0 == 1:
                batch_pred = self.point_sf(X.unsqueeze(0)).view(1, -1)
                layout = {}
            else:
                batch_pred = self.div_forward_ragged(X, off, max_len)
                layout = dict(offsets=off, max_len=max_len)
            if check and self.stop_training(batch_pred):
                stop_training = True
                break
            losses.append(self.div_custom_loss_function(batch_pred, sp.rele.select(q0, q1), presort=True,
                                                        **layout).detach())
        total = float(torch.stack(losses).double().sum()) if losses else 0.0
        epoch_loss = torch.tensor([total / len(train_data)], device=self.device)
        return epoch_loss, stop_training

    def div_train_op(self, q_repr, doc_reprs, q_doc_rele_mat, **kwargs):
        """ranker.py:659-670: one query's step from host or device tensors (div_train uses the packed split)."""
        stop_training = False
        batch_pred = self.div_forward(q_repr.to(self.device), doc_reprs.to(self.device))
        if 'epoch_k' in kwargs and kwargs['epoch_k'] is not None and kwargs['epoch_k'] % self.stop_check_freq == 0:
            stop_training = self.stop_training(batch_pred)
        rele = ops.SubtopicRele.pack([q_doc_rele_mat], self.device)
        return self.div_custom_loss_function(batch_pred, rele, **kwargs), stop_training

    def div_custom_loss_function(self, batch_preds, q_doc_rele_mat, **kwargs):
        pass

    # ---- evaluation --------------------------------------------------------------------------------------------- #
    def _metrics(self, data, ks, max_label=None, return_order=False):
        """One scorer forward and one metric launch over the whole split -> (split, andcg, err_ia, nerr_ia, flags
        [, order]) on the device."""
        self.eval_mode()
        sp = self._split(data)
        preds = self.split_keys(sp)
        res = ops.srd_metrics_at_ks(preds, sp.rele, ks, max_label=1.0 if max_label is None else max_label,
                                    offsets=sp.offsets, max_len=sp.max_len, return_order=return_order)
        return (sp, *res)

    @staticmethod
    def _average(vals, mask):
        """sum over the counted queries / their number: one device-to-host copy."""
        m = mask.to(vals.dtype).unsqueeze(1)
        cnt = mask.sum()
        return (torch.sum(vals * m, dim=0) / cnt).cpu()

    def _at_k(self, which, test_data, k, max_label=None):
        """alpha_ndcg_at_k / err_ia_at_k / nerr_ia_at_k (ranker.py:265-411): queries with sum(R) < 1 or fewer than k
        documents are skipped."""
        if which != 1:
            assert getattr(test_data, 'presort', True) is True
        if which != 0:
            assert max_label is not None
        sp, andcg, err, nerr, flags = self._metrics(test_data, [k], max_label)
        mask = ((flags & 1) != 0) & (sp.lens >= k)
        return self._average((andcg, err, nerr)[which], mask)

    def alpha_ndcg_at_k(self, test_data=None, k=5, device='cpu'):
        return self._at_k(0, test_data, k)

    def err_ia_at_k(self, test_data=None, k=5, max_label=None, device='cpu'):
        return self._at_k(1, test_data, k, max_label)

    def nerr_ia_at_k(self, test_data=None, k=5, max_label=None, device='cpu'):
        return self._at_k(2, test_data, k, max_label)

    def alpha_ndcg_at_ks(self, test_data=None, ks=[1, 5, 10], device='cpu'):
        """ranker.py:303-330: only queries with sum(R) < 1 are skipped; a cutoff beyond a list's length counts 0."""
        assert getattr(test_data, 'presort', True) is True
        sp, andcg, _, _, flags = self._metrics(test_data, ks)
        return self._average(andcg, (flags & 1) != 0)

    def srd_performance_at_ks(self, test_data=None, ks=[1, 5, 10], max_label=None, device='cpu',
                              generate_div_run=False, dir=None, fold_k=None, need_per_q_andcg=False):
        """ranker.py:413-475: average alpha-nDCG, ERR-IA and nERR-IA at ks over the queries with sum(R) > 0."""
        assert getattr(test_data, 'presort', True) is True
        assert max_label is not None
        res = self._metrics(test_data, ks, max_label, return_order=generate_div_run)
        sp, andcg, err, nerr, flags = res[:5]
        mask = (flags & 2) != 0
        m = mask.to(torch.float32).unsqueeze(1)
        sums = torch.stack([torch.sum(v * m, dim=0) for v in (andcg, err, nerr)])
        packed = torch.cat([sums.reshape(-1), mask.to(torch.float32), andcg.reshape(-1)]).cpu()
        nk, Q = len(ks), len(sp)
        num_queries = float(packed[3 * nk: 3 * nk + Q].sum())
        avgs = [packed[i * nk:(i + 1) * nk] / num_queries for i in range(3)]
        if generate_div_run:
            order = res[5].cpu().numpy()
            counted = packed[3 * nk: 3 * nk + Q].numpy()
            with open(dir + '/fold_run.txt', 'w') as fold_run:
                for q in range(Q):
                    if not counted[q]:
                        continue
                    o0, o1 = sp.offsets_host[q], sp.offsets_host[q + 1]
                    num_docs = int(o1 - o0)
                    for i in range(num_docs):
                        doc = sp.perm_docs[q][int(order[o0 + i])]
                        fold_run.write(' '.join([str(sp.qids[q]), 'Q0', doc, str(i + 1), str(num_docs - i),
                                                 'Fold' + str(fold_k) + "\n"]))
        if need_per_q_andcg:
            per_q = packed[3 * nk + Q:].reshape(Q, nk)
            counted = packed[3 * nk: 3 * nk + Q]
            return (*avgs, [per_q[q:q + 1] for q in range(Q) if counted[q]])
        return tuple(avgs)

    def div_validation(self, vali_data=None, vali_metric=None, k=5, max_label=None, device='cpu'):
        """diversity_ranker.py:58-64."""
        if 'aNDCG' == vali_metric:
            return self.alpha_ndcg_at_k(test_data=vali_data, k=k, device=device)
        elif 'nERR-IA' == vali_metric:
            return self.nerr_ia_at_k(test_data=vali_data, k=k, max_label=max_label, device=device)
        else:
            raise NotImplementedError

    # ---- modes and checkpoints ---------------------------------------------------------------------------------- #
    def eval_mode(self):
        if 'pointsf' == self.sf_id:
            return PointNeuralRanker.eval_mode(self)
        for part in self.list_sf.values():
            part.eval()

    def train_mode(self):
        if 'pointsf' == self.sf_id:
            return PointNeuralRanker.train_mode(self)
        for part in self.list_sf.values():
            part.train(mode=True)

    def save(self, dir, name):
        """pointsf: the scorer's state_dict; listsf: {'encoder': ..., 'uni_sf': ...} (div_list_ranker.py:100-105)."""
        if 'pointsf' == self.sf_id:
            return PointNeuralRanker.save(self, dir, name)
        if not os.path.exists(dir):
            os.makedirs(dir)
        torch.save({'encoder': self.list_sf['encoder'].state_dict(), 'uni_sf': self.list_sf['uni_sf'].state_dict()},
                   dir + name)

    def load(self, file_model, **kwargs):
        """The driver loads with context='cpu_gpu' and no device (ltr_diversification.py:296-302)."""
        device = kwargs.get('device') or self.device
        if 'pointsf' == self.sf_id:
            self.point_sf.load_state_dict(torch.load(file_model, map_location=device))
            return
        checkpoint = torch.load(file_model, map_location=device)
        self.list_sf['encoder'].load_state_dict(checkpoint['encoder'])
        self.list_sf['uni_sf'].load_state_dict(checkpoint['uni_sf'])

    def uniform_eval_setting(self, **kwargs):
        pass
