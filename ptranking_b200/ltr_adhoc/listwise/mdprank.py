"""MDPRank (mirror of ptranking/ltr_adhoc/listwise/mdprank.py:13-79).

One fused kernel per batch samples a Plackett-Luce ranking per query (Gumbel-perturbed sort), forms the discounted
returns of its rewards and the REINFORCE loss and gradient (ptrb200_mdprank_fwd_bwd).  Unlike the reference it takes
any number of queries per batch, ragged batches included (the batch loss is the sum over queries), and clamps top_k
to each list's length.
"""
from ...base.adhoc_ranker import AdhocNeuralRanker
from ... import ops
from ..._lib import MDP_DISTRIBUTIONS


class MDPRank(AdhocNeuralRanker):
    def __init__(self, sf_para_dict=None, model_para_dict=None, gpu=False, device=None):
        # checked before the device, so a bad configuration is reported as such on any machine
        if model_para_dict['distribution'] not in MDP_DISTRIBUTIONS:
            raise NotImplementedError(f"MDPRank distribution={model_para_dict['distribution']!r} is not one of "
                                      f"{sorted(MDP_DISTRIBUTIONS)}")
        super().__init__(id='MDPRank', sf_para_dict=sf_para_dict, gpu=gpu, device=device)
        self.gamma = model_para_dict['gamma']
        self.top_k = model_para_dict['top_k']
        self.temperature = model_para_dict['temperature']
        self.distribution = model_para_dict['distribution']  # 'PL', 'STPL'

    def custom_loss_function(self, batch_preds, batch_std_labels, **kwargs):
        """Sum over the queries of the policy-gradient loss of one sampled ranking each (mdprank.py:24-79).  The draw
        comes from the kernel's counter-based generator (the reference calls torch.multinomial / torch.rand);
        ``perm=`` (int [B,n], PL only) injects the ordering and ``unif=`` the uniforms behind the Gumbel noise."""
        assert 'presort' in kwargs and kwargs['presort'] is True  # aiming for direct usage of ideal ranking
        batch_loss = ops.rank_loss('MDPRank', batch_preds, batch_std_labels, distribution=self.distribution,
                                   top_k=self.top_k, gamma=float(self.gamma), temperature=float(self.temperature),
                                   perm=kwargs.get('perm'), unif=kwargs.get('unif'), **self.ragged_kwargs(kwargs))
        self.backward_and_step(batch_loss)
        return batch_loss
