"""WassRank (mirror of ptranking/ltr_adhoc/listwise/wassrank/wassRank.py:22-86), mode 'SinkhornOT'.

The whole loss -- cost matrix, softmax histograms, Sinkhorn iterations, loss and the reference's gradient -- is one
fused kernel per batch (ptrb200_wassrank_fwd_bwd).  Unlike the reference it runs at any batch size and on ragged
batches (every query gets its own cost matrix; the loss is the mean over queries), and it iterates in the log domain, so
it stays finite where exp(-C/lam) underflows in fp32.
"""
import math

from ...base.adhoc_ranker import AdhocNeuralRanker
from ... import ops
from ..._lib import WASS_COST_TYPES

# WassRankParameter.default_para_dict, wassRank.py:97-104
DEFAULT_WASS_PARA = dict(model_id='WassRank', mode='SinkhornOT', sh_itr=20, lam=0.1, smooth_type='ST', norm_type='BothST',
                         cost_type='eg', non_rele_gap=100, var_penalty=math.e, gain_base=4)


def check_wass_para_dict(wass_para_dict):
    """-> the settings the kernel runs, or an error naming the unsupported one."""
    para = dict(DEFAULT_WASS_PARA)
    para.update(wass_para_dict or {})
    if para['mode'] == 'EntropicOT':
        raise NotImplementedError("WassRank mode='EntropicOT' is not supported: it differentiates through a Sinkhorn loop "
                                  "whose early stop reads the error of the whole batch back to the host; use mode='SinkhornOT'")
    if para['mode'] != 'SinkhornOT':
        raise NotImplementedError(f"WassRank mode={para['mode']!r} is not supported (the reference knows 'SinkhornOT' and 'EntropicOT')")
    if para['smooth_type'] == 'NG':
        raise NotImplementedError("WassRank smooth_type='NG' is not supported: its batch-wide minimum shift gives the lowest "
                                  "scored document zero mass, so the loss takes log 0; use smooth_type='ST'")
    if para['smooth_type'] != 'ST' or para['norm_type'] != 'BothST':
        raise NotImplementedError(f"WassRank supports smooth_type='ST' with norm_type='BothST', got "
                                  f"{para['smooth_type']!r} / {para['norm_type']!r}")
    if para['cost_type'] not in WASS_COST_TYPES:
        raise NotImplementedError(f"WassRank cost_type={para['cost_type']!r} is not one of {sorted(WASS_COST_TYPES)}")
    if not float(para['lam']) > 0.0 or int(para['sh_itr']) < 0:
        raise ValueError(f"WassRank needs lam > 0 and sh_itr >= 0, got lam={para['lam']} sh_itr={para['sh_itr']}")
    return para


class WassRank(AdhocNeuralRanker):
    def __init__(self, sf_para_dict=None, wass_para_dict=None, dict_cost_mats=None, dict_std_dists=None, gpu=False, device=None):
        # settings are checked before the device, so a bad configuration is reported as such on any machine
        self.wass_para_dict = check_wass_para_dict(wass_para_dict)
        super().__init__(id='WassRank', sf_para_dict=sf_para_dict, gpu=gpu, device=device)
        # dict_cost_mats / dict_std_dists only cache what the kernel recomputes from the labels: accepted, not used.
        # The histogram of the predictions is softmax(scores) as given: the reference's rescaling by the largest label
        # (wasserstein_cost_mat.py:197-199) never runs there, because its get_tl_af returns None (adhoc_ranker.py:83-87).
        self.dict_cost_mats, self.dict_std_dists = dict_cost_mats, dict_std_dists

    def custom_loss_function(self, batch_preds, batch_std_labels, **kwargs):
        """Mean over the batch of the queries' Sinkhorn transport costs; the scorer receives the reference's gradient."""
        p = self.wass_para_dict
        batch_loss = ops.rank_loss('WassRank', batch_preds, batch_std_labels, cost_type=p['cost_type'], lam=float(p['lam']),
                                   sh_itr=int(p['sh_itr']), non_rele_gap=float(p['non_rele_gap']),
                                   var_penalty=float(p['var_penalty']), gain_base=float(p['gain_base']),
                                   **self.ragged_kwargs(kwargs))
        self.backward_and_step(batch_loss)
        return batch_loss
