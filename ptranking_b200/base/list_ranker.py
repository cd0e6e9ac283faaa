"""Multi-head self-attention list ranker -- mirror of ptranking/base/list_ranker.py (Encoder :53, EncoderLayer :87,
SublayerConnection :118, LayerNorm :152, MultiheadAttention :176, PositionwiseFeedForward :256,
ListNeuralRanker :280-402).  Module names follow the reference so its three-part checkpoint
(``head_ffnns`` / ``encoder`` / ``tail_ffnns`` state_dicts, list_ranker.py:390-402) loads unchanged; every
tensor operation goes to the CUDA kernels through ptranking_b200.ops."""
from __future__ import annotations

import copy
import os

import torch
import torch.nn as nn

from .. import ops
from .ranker import NeuralRanker
from .utils import get_stacked_FFNet

Encoder_Type = ['DASALC', 'AllRank', 'AttnDIN']


class LayerNorm(nn.Module):
    """a_2 (x - mean) / (std + eps) + b_2 with the unbiased std (list_ranker.py:152-174)."""

    def __init__(self, hid_dim, eps=1e-6):
        super().__init__()
        self.a_2 = nn.Parameter(torch.ones(hid_dim))
        self.b_2 = nn.Parameter(torch.zeros(hid_dim))
        self.eps = eps

    def forward(self, x):
        return ops.layernorm_ref(x, self.a_2, self.b_2, self.eps)


class MultiheadAttention(nn.Module):
    """list_ranker.py:176-254: Q/K/V projections, softmax(QK^T/sqrt(d)) with dropout, .V, output projection."""

    def __init__(self, hid_dim, n_heads, dropout=0.1, device=None):
        super().__init__()
        assert hid_dim % n_heads == 0
        self.hid_dim, self.n_heads, self.p = hid_dim, n_heads, dropout
        self.w_q, self.w_k, self.w_v = nn.Linear(hid_dim, hid_dim), nn.Linear(hid_dim, hid_dim), nn.Linear(hid_dim, hid_dim)
        self.fc = nn.Linear(hid_dim, hid_dim, bias=True)

    def projection_parameters(self):
        """Order in which the ranker lays this block out in its flat parameter buffer: the three projection weights
        side by side (then their biases), so that forward() can treat them as ONE [3*hid, hid] matrix in place."""
        return [self.w_q.weight, self.w_k.weight, self.w_v.weight, self.w_q.bias, self.w_k.bias, self.w_v.bias,
                self.fc.weight, self.fc.bias]

    def forward(self, x):
        p = self.p if self.training else 0.0
        if ops.attention_impl() in ("tc", "tc_tf32") and os.environ.get("PTRANKING_B200_FUSED_QKV", "1") == "1":
            # Q|K|V = x [Wq;Wk;Wv]^T + [bq;bk;bv]: one hid -> 3*hid contraction (column for column the reference's three,
            # list_ranker.py:233-235), read in place by the attention kernels; its backward is one data-gradient and
            # one weight-gradient contraction instead of three each plus two tensor additions
            W = ops.adjacent_rows(self.w_q.weight, self.w_k.weight, self.w_v.weight)
            b = ops.adjacent_rows(self.w_q.bias, self.w_k.bias, self.w_v.bias)
            ctx = ops.attention_packed(ops.linear(x, W, b), self.n_heads, p)
        else:
            Q = ops.linear(x, self.w_q.weight, self.w_q.bias)
            K = ops.linear(x, self.w_k.weight, self.w_k.bias)
            V = ops.linear(x, self.w_v.weight, self.w_v.bias)
            ctx = ops.attention(Q, K, V, self.n_heads, p)
        return ops.linear(ctx, self.fc.weight, self.fc.bias)


class PositionwiseFeedForward(nn.Module):
    """w2(dropout(relu(w1 x))) (list_ranker.py:256-277)."""

    def __init__(self, num_features, hid_dim, dropout=0.1):
        super().__init__()
        self.w1, self.w2, self.p = nn.Linear(num_features, hid_dim), nn.Linear(hid_dim, num_features), dropout

    def forward(self, x):
        h = ops.dropout(ops.relu(ops.linear(x, self.w1.weight, self.w1.bias)), self.p, self.training)
        return ops.linear(h, self.w2.weight, self.w2.bias)


class SublayerConnection(nn.Module):
    """list_ranker.py:118-149."""

    def __init__(self, hid_dim, encoder_type=None, dropout=None):
        super().__init__()
        self.encoder_type = encoder_type
        self.norm = LayerNorm(hid_dim=hid_dim)
        self.p = dropout if 'AllRank' == encoder_type else 0.0

    def forward(self, x, sublayer):
        if 'AllRank' == self.encoder_type:
            return ops.add(x, ops.dropout(sublayer(self.norm(x)), self.p, self.training))
        if 'DASALC' == self.encoder_type:
            return self.norm(sublayer(x))
        if 'AttnDIN' == self.encoder_type:
            return self.norm(ops.add(x, sublayer(x)))
        raise NotImplementedError


class EncoderLayer(nn.Module):
    """list_ranker.py:87-115."""

    def __init__(self, hid_dim, mhsa, encoder_type=None, fc=None, dropout=None):
        super().__init__()
        self.mhsa, self.hid_dim, self.encoder_type = mhsa, hid_dim, encoder_type
        if 'AllRank' == encoder_type:
            self.fc = fc
            self.sublayer_cont = nn.ModuleList([copy.deepcopy(SublayerConnection(hid_dim, encoder_type, dropout)) for _ in range(2)])
        elif encoder_type in ['AttnDIN', 'DASALC']:
            self.sublayer_cont = SublayerConnection(hid_dim=hid_dim, encoder_type=encoder_type)
        else:
            raise NotImplementedError

    def forward(self, x):
        if 'AllRank' == self.encoder_type:
            x = self.sublayer_cont[0](x, self.mhsa)
            return self.sublayer_cont[1](x, self.fc)
        return self.sublayer_cont(x, self.mhsa)


class Encoder(nn.Module):
    """N clones of one EncoderLayer -- the clones start from identical weights, as in make_clones
    (list_ranker.py:48-50, 53-85)."""

    def __init__(self, layer, num_layers, encoder_type=None):
        super().__init__()
        self.encoder_type = encoder_type
        self.layers = nn.ModuleList([copy.deepcopy(layer) for _ in range(num_layers)])
        if 'AllRank' == encoder_type:
            self.norm = LayerNorm(layer.hid_dim)

    def forward(self, x):
        for layer in self.layers:
            x = layer(x)
        return self.norm(x) if 'AllRank' == self.encoder_type else x


def encoder_parameters(encoder):
    """The encoder's parameters with each attention block's projection weights side by side
    (MultiheadAttention.projection_parameters), so that a flat parameter buffer holds them as one [3*hid, hid] matrix."""
    enc, seen = [], set()
    for m in encoder.modules():
        if isinstance(m, MultiheadAttention):
            for p in m.projection_parameters():
                if id(p) not in seen:
                    seen.add(id(p)); enc.append(p)
    return enc + [p for p in encoder.parameters() if id(p) not in seen]


class ListNeuralRanker(NeuralRanker):
    """Permutation-equivariant ranker: head FFN, MHSA encoder, tail FFN (list_ranker.py:280-402)."""

    def __init__(self, id='ListNeuralRanker', sf_para_dict=None, weight_decay=1e-3, gpu=False, device=None):
        super().__init__(id=id, sf_para_dict=sf_para_dict, weight_decay=weight_decay, gpu=gpu, device=device)
        self.encoder_type = self.sf_para_dict[self.sf_para_dict['sf_id']]['encoder_type']

    def init(self):
        self.list_sf = self.config_list_neural_scoring_function()
        self.config_optimizer()

    def config_list_neural_scoring_function(self):
        return self.ini_listsf(**self.sf_para_dict[self.sf_para_dict['sf_id']])

    def get_parameters(self):
        """Same set as the reference (list_ranker.py:297-301); inside the encoder each attention block's projection
        weights are listed side by side (encoder_parameters) -- the order only decides the layout of the flat parameter /
        gradient buffers, checkpoints are per-module state_dicts."""
        return list(self.list_sf['head_ffnns'].parameters()) + encoder_parameters(self.list_sf['encoder']) + \
            list(self.list_sf['tail_ffnns'].parameters())

    def ini_listsf(self, num_features=None, ff_dims=[128, 256, 512], out_dim=1, AF='R', TL_AF='GE', apply_tl_af=False,
                   BN=True, bn_type=None, bn_affine=False, n_heads=2, encoder_layers=3, dropout=0.1, encoder_type=None):
        """list_ranker.py:303-349.  The head net always ends in AF (:313); the tail net is built without the
        configured dropout and keeps the factory default 0.1 (:340-341, SURVEY B10)."""
        F = num_features
        head_ffnns = get_stacked_FFNet(ff_dims=[F, *ff_dims, F], AF=AF, TL_AF=AF, apply_tl_af=True, dropout=dropout,
                                       BN=BN, bn_type=bn_type, bn_affine=bn_affine, device=self.device)
        mhsa = MultiheadAttention(hid_dim=F, n_heads=n_heads, dropout=dropout, device=self.device)
        if 'AllRank' == encoder_type:
            fc = PositionwiseFeedForward(F, hid_dim=F, dropout=dropout)
            layer = EncoderLayer(hid_dim=F, mhsa=copy.deepcopy(mhsa), encoder_type=encoder_type, fc=fc, dropout=dropout)
        elif encoder_type in ('DASALC', 'AttnDIN'):
            layer = EncoderLayer(hid_dim=F, mhsa=copy.deepcopy(mhsa), encoder_type=encoder_type)
        else:
            raise NotImplementedError
        encoder = Encoder(layer=layer, num_layers=encoder_layers, encoder_type=encoder_type)
        tail_ffnns = get_stacked_FFNet(ff_dims=[F, *ff_dims, out_dim], AF=AF, TL_AF=TL_AF, apply_tl_af=apply_tl_af,
                                       BN=BN, bn_type=bn_type, bn_affine=bn_affine, device=self.device)
        return {'head_ffnns': head_ffnns.to(self.device), 'encoder': encoder.to(self.device),
                'tail_ffnns': tail_ffnns.to(self.device)}

    def forward(self, batch_q_doc_vectors):
        """[B,n,F] -> [B,n] (list_ranker.py:351-378).  bf16 features are upcast to fp32 here: the encoder and the
        DASALC / AttnDIN glue consume X in fp32 (only the pointwise scorer reads bf16 features natively)."""
        X = batch_q_doc_vectors
        if X.dtype != torch.float32:
            X = X.float()
        head, enc, tail = self.list_sf['head_ffnns'], self.list_sf['encoder'], self.list_sf['tail_ffnns']
        if 'AllRank' == self.encoder_type:
            z = enc(head(X))
        elif 'DASALC' == self.encoder_type:
            z = ops.latent_cross(enc(X), head(X))
        elif 'AttnDIN' == self.encoder_type:
            z = ops.add(enc(head(X)), X)
        else:
            raise NotImplementedError
        return torch.squeeze(tail(z), dim=2)

    def forward_ragged(self, flat_q_doc_vectors, offsets, max_len, buckets=None):
        """[total_docs, F] + int32 offsets[B+1] -> flat scores [total_docs] for lists of different lengths (the reference can
        only batch equal-length lists, data_utils.py:683-742).  The batch is padded on the device, the attention masks
        every query's padded keys (probability exactly 0), all other layers are row-wise, and the scores of the real
        documents are gathered back -- so each query sees exactly what it would see alone.  With ``buckets``
        (data.RaggedBatches: the batch sorted by length and cut into length classes) every class is padded to ITS longest
        list only.  Batch- or list-level normalisation in the head / tail nets would mix padding into its statistics and
        is refused."""
        cfg = self.sf_para_dict[self.sf_para_dict['sf_id']]
        if cfg.get('BN', True):
            raise NotImplementedError("ragged batches through the list scorer need BN=False (the listsf default of the drop-in run)")
        X = flat_q_doc_vectors
        total = X.shape[0]
        offs = offsets.to(device=X.device, dtype=torch.int32).contiguous()
        B = offs.numel() - 1
        classes = [(int(q0), int(q1), max(int(ml), 1)) for q0, q1, ml in buckets if int(q1) > int(q0)] if buckets else []
        if not classes:
            classes = [(0, B, max(int(max_len), 1))]
        if classes[0][0] != 0 or classes[-1][1] != B or any(a[1] != b[0] for a, b in zip(classes, classes[1:])):
            raise ValueError("buckets must cover the queries of the batch in order")
        padded = []
        for q0, q1, nmax in classes:
            sub = offs[q0: q1 + 1]                      # absolute prefix offsets: the kernels index the whole flat batch
            with ops.key_lens_context((sub[1:] - sub[:-1]).contiguous()):
                padded.append(self.forward(ops.pad_lists(X, sub, nmax)).contiguous())     # [q1 - q0, nmax]
        return ops.unpad_buckets(padded, offs, total, [c[0] for c in classes])

    def eval_mode(self):
        for part in self.list_sf.values():
            part.eval()

    def train_mode(self):
        for part in self.list_sf.values():
            part.train(mode=True)

    def save(self, dir, name):
        if not os.path.exists(dir):
            os.makedirs(dir)
        torch.save({k: v.state_dict() for k, v in self.list_sf.items()}, dir + name)

    def load(self, file_model, device=None, **kwargs):
        checkpoint = torch.load(file_model, map_location=device)
        for k in ('head_ffnns', 'encoder', 'tail_ffnns'):
            self.list_sf[k].load_state_dict(checkpoint[k])
