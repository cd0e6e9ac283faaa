"""DALETOR (mirror of ptranking/ltr_diversification/score_and_sort/daletor.py:43-71).

One fused kernel per batch computes the alpha-DCG loss of the sigmoid rank approximation and its gradient for every
query (ptrb200_daletor_fwd_bwd); the reference builds [m, n, n] temporaries per query and differentiates them with
autograd.  With the reference's one query per step the two agree; ``queries_per_step`` > 1 sums the queries' losses.
"""
from ..base.diversity_ranker import DiversityNeuralRanker
from ... import ops


class DALETOR(DiversityNeuralRanker):
    """Le Yan, Zhen Qin, Rama Kumar Pasumarthi, Xuanhui Wang, Mike Bendersky.  Diversification-Aware Learning to Rank
    using Distributed Representation.  The Web Conference 2021 (WWW)."""

    def __init__(self, sf_para_dict=None, model_para_dict=None, gpu=False, device=None):
        super().__init__(id='DALETOR', sf_para_dict=sf_para_dict, gpu=gpu, device=device)
        self.rt = model_para_dict['rt']
        self.top_k = model_para_dict['top_k']

    def div_custom_loss_function(self, batch_preds, q_doc_rele_mat, **kwargs):
        """alphaDCG_as_a_loss (daletor.py:22-40) with alpha = 0.5, as the reference calls it.  ``q_doc_rele_mat``: the
        batch's ops.SubtopicRele; ``offsets``/``max_len`` for a ragged batch of several queries."""
        assert 'presort' in kwargs and kwargs['presort'] is True  # aiming for directly optimising alpha-nDCG over top-k
        preds = batch_preds if kwargs.get('offsets') is not None else batch_preds.view(1, -1)
        batch_loss, _ = ops.daletor_loss(preds, q_doc_rele_mat, rt=float(self.rt), top_k=self.top_k, alpha=0.5,
                                         offsets=kwargs.get('offsets'), max_len=kwargs.get('max_len'))
        self.backward_and_step(batch_loss)
        return batch_loss
