"""The diversification list scorer (mirror of ptranking/ltr_diversification/base/div_list_ranker.py).

An MHSA encoder of width 3F over each query's [q, d, q*d] rows (no head net, no tail net), then a univariate stacked
FF net ``uni_sf`` over [q, d, q*d, enc] (width 6F) with BN statistics per query.  The reference runs one query per
call.  Here a ragged batch -- a training step of several queries, or a whole split -- is cut into length classes: each
class is padded to its longest list (ops.pad_lists_pitched), goes through the encoder with its padded keys masked, and
one launch per class writes the class's rows of the uni_sf input (ops.div_list_concat).  uni_sf then scores all flat
rows in one call, its per-query BN keeping the reference's one-query statistics.
"""
from __future__ import annotations

import copy

import numpy as np
import torch

from ... import ops
from ...base.list_ranker import Encoder, EncoderLayer, Encoder_Type, MultiheadAttention, PositionwiseFeedForward, \
    encoder_parameters
from ...base.utils import StackedFFNet

# Memory budget of one chunk of a length class: its fp32 [B*H, n, n] attention probabilities stay below this many
# bytes (a longer list than the budget allows still goes alone).  Evaluation frees each chunk's attention before the
# next one; a training step keeps every chunk's for the backward pass.
ATTN_BUDGET_BYTES = 256 << 20


def check_listsf_config(cfg):
    """Refuse a listsf dict this scorer does not build, before any device is touched.  The reference raises
    NotImplementedError for an unknown encoder_type and KeyError for a missing one; both raise NotImplementedError
    here."""
    enc = cfg.get('encoder_type')
    if enc not in Encoder_Type:
        raise NotImplementedError(f"the diversification list scorer has no encoder_type {enc!r} "
                                  f"(one of {', '.join(Encoder_Type)})")
    if cfg.get('BN', True) and cfg.get('bn_type') != 'BN':
        # LTRBatchNorm2 on the reference's 2-D [n, C] uni_sf input would normalise over features, not documents
        raise NotImplementedError("the diversification list scorer's uni_sf supports BN=False or bn_type='BN' only")


def length_classes(lens, n_heads, budget=ATTN_BUDGET_BYTES):
    """Cut the queries with documents into length classes -> [(query indices, padded length)].  Longest first: a class
    takes the longest remaining list n and then, in descending length, lists longer than n / 2 (so padding at most
    doubles a class's rows), while its [B*H, n, n] fp32 attention tensor stays within ``budget`` bytes."""
    lens = np.asarray(lens, dtype=np.int64)
    order = [int(q) for q in np.argsort(-lens, kind='stable') if lens[q] > 0]
    out, i = [], 0
    while i < len(order):
        n = int(lens[order[i]])
        cap = max(1, int(budget) // (4 * n_heads * n * n))
        j = i + 1
        while j < len(order) and j - i < cap and 2 * int(lens[order[j]]) > n:
            j += 1
        out.append((order[i:j], n))
        i = j
    return out


class ListPlan:
    """A ragged batch's layout for the list scorer, on the device: int32 prefix offsets, and per length class its
    int32 query indices, the key lengths to mask (None when every list of the class fills it) and its padded length."""

    def __init__(self, offsets_host, n_heads, budget, device):
        o = np.asarray(offsets_host, dtype=np.int64)
        o = o - o[0]
        lens = o[1:] - o[:-1]
        self.offsets = torch.from_numpy(o.astype(np.int32)).to(device)
        self.max_len = max(int(lens.max(initial=0)), 1)
        self.classes = []
        for qs, n in length_classes(lens, n_heads, budget):
            qidx = torch.tensor(qs, dtype=torch.int32).to(device)
            klens = None if all(int(lens[q]) == n for q in qs) else \
                torch.tensor([int(lens[q]) for q in qs], dtype=torch.int32).to(device)
            self.classes.append((qidx, klens, n))


class DivListNeuralRanker:
    """The listsf half of DiversityNeuralRanker (which dispatches on sf_id as the reference's does)."""

    def ini_listsf(self, num_features=None, n_heads=2, encoder_layers=2, dropout=0.1, encoder_type=None,
                   ff_dims=[256, 128, 64], out_dim=1, AF='R', TL_AF='GE', apply_tl_af=False, BN=True, bn_type=None,
                   bn_affine=False):
        """div_list_ranker.py:20-59.  uni_sf is built without the configured dropout and keeps the factory default 0.1
        (SURVEY B10); its BN normalises each query over its own documents, as LTRBatchNorm does on the reference's
        one-query [n, 6F] input."""
        W = 3 * num_features
        mhsa = MultiheadAttention(hid_dim=W, n_heads=n_heads, dropout=dropout, device=self.device)
        if 'AllRank' == encoder_type:
            fc = PositionwiseFeedForward(W, hid_dim=W, dropout=dropout)
            layer = EncoderLayer(hid_dim=W, mhsa=copy.deepcopy(mhsa), encoder_type=encoder_type, fc=fc, dropout=dropout)
        elif encoder_type in ('DASALC', 'AttnDIN'):
            layer = EncoderLayer(hid_dim=W, mhsa=copy.deepcopy(mhsa), encoder_type=encoder_type)
        else:
            raise NotImplementedError
        encoder = Encoder(layer=layer, num_layers=encoder_layers, encoder_type=encoder_type)
        uni_sf = StackedFFNet([2 * W, *ff_dims, out_dim], AF=AF, TL_AF=TL_AF, apply_tl_af=apply_tl_af, dropout=0.1,
                              BN=BN, bn_type=bn_type, bn_affine=bn_affine, device=self.device,
                              bn_per_query=bool(BN) and bn_type == 'BN', pad_output=True)
        return {'encoder': encoder.to(self.device), 'uni_sf': uni_sf.to(self.device)}

    def list_parameters(self):
        """div_list_ranker.py:87-90: the encoder (projection weights side by side, see encoder_parameters), then
        uni_sf."""
        return encoder_parameters(self.list_sf['encoder']) + list(self.list_sf['uni_sf'].parameters())

    def list_plan(self, offsets_host):
        return ListPlan(offsets_host, self.sf_para_dict['listsf'].get('n_heads', 2), self.attn_budget_bytes, self.device)

    def list_scores(self, X, plan):
        """[rows, 3F] encoder input of a ragged batch laid out by ``plan`` -> flat scores [rows]."""
        qidxs, blocks = [], []
        for qidx, klens, n in plan.classes:
            P = ops.pad_lists_pitched(X, plan.offsets, qidx, n)
            with ops.key_lens_context(klens):
                blocks.append(self.list_sf['encoder'](P))
            qidxs.append(qidx)
        Z = ops.div_list_concat(X, plan.offsets, qidxs, blocks)
        return self.list_sf['uni_sf'](Z, offsets=plan.offsets, max_len=plan.max_len).view(-1)

    def list_div_forward(self, q_repr, doc_reprs):
        """div_list_ranker.py:61-85: q_repr [1,F], doc_reprs [n,F] -> [1,n]."""
        n = doc_reprs.size(0)
        X = ops.div_list_features(q_repr.reshape(1, -1), doc_reprs.reshape(n, -1), offsets=self._one_query_offsets(n),
                                  max_len=n)
        return self.list_scores(X, self.list_plan([0, n])).view(1, -1)

    def _one_query_offsets(self, n):
        return torch.tensor([0, n], dtype=torch.int32).to(self.device)
