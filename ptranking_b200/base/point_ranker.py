"""Pointwise MLP ranker (mirror of ptranking/base/point_ranker.py:9-74)."""
from __future__ import annotations

import os

import torch

from .ranker import NeuralRanker
from .utils import get_stacked_FFNet


class PointNeuralRanker(NeuralRanker):
    """Scores every document of a query independently with one stacked feed-forward net."""

    def __init__(self, id='PointNeuralRanker', sf_para_dict=None, weight_decay=1e-3, gpu=False, device=None):
        super().__init__(id=id, sf_para_dict=sf_para_dict, weight_decay=weight_decay, gpu=gpu, device=device)

    def init(self):
        self.point_sf = self.config_point_neural_scoring_function()
        self.config_optimizer()
        # the scorer is a single fused op whose backward overwrites every parameter gradient: let it write
        # straight into the flat gradient bucket (no per-tensor accumulate kernels, no zero fill)
        self.point_sf.write_through_grads = True
        # (a zero-padded output layer, StackedFFNet._pad_out, hands its gradients to autograd instead: zero the bucket)
        self.grad_bucket_overwritten = not self.point_sf._pad_out

    def config_point_neural_scoring_function(self):
        point_sf = self.ini_pointsf(**self.sf_para_dict[self.sf_para_dict['sf_id']])
        return point_sf.to(self.device)

    def get_parameters(self):
        return self.point_sf.parameters()

    def ini_pointsf(self, num_features=None, h_dim=100, out_dim=1, num_layers=3, AF='R', TL_AF='S', apply_tl_af=False,
                    BN=True, bn_type=None, bn_affine=False, dropout=0.1):
        """point_ranker.py:30-42: widths [F, h*num_layers, out]."""
        ff_dims = [num_features] + [h_dim] * num_layers + [out_dim]
        return get_stacked_FFNet(ff_dims=ff_dims, AF=AF, TL_AF=TL_AF, apply_tl_af=apply_tl_af, dropout=dropout,
                                 BN=BN, bn_type=bn_type, bn_affine=bn_affine, device=self.device)

    def forward(self, batch_q_doc_vectors):
        """[B,n,F] -> [B,n] (point_ranker.py:45-55)."""
        num_docs = batch_q_doc_vectors.size(1)
        return self.point_sf(batch_q_doc_vectors).view(-1, num_docs)

    def forward_ragged(self, flat_q_doc_vectors, offsets, max_len, buckets=None):
        """[total_docs, F] -> [total_docs]: the pointwise scorer acts per document, so a ragged batch is one long list
        to it; only per-query normalisation (BN2) needs the offsets (length classes are of no use here)."""
        return self.point_sf(flat_q_doc_vectors, offsets=offsets, max_len=max_len).view(-1)

    def eval_mode(self):
        self.point_sf.eval()

    def train_mode(self):
        self.point_sf.train(mode=True)

    def save(self, dir, name):
        if not os.path.exists(dir):
            os.makedirs(dir)
        torch.save(self.point_sf.state_dict(), dir + name)

    def load(self, file_model, **kwargs):
        device = kwargs['device']
        self.point_sf.load_state_dict(torch.load(file_model, map_location=device))

    def get_tl_af(self):
        return self.sf_para_dict[self.sf_para_dict['sf_id']]['TL_AF']
