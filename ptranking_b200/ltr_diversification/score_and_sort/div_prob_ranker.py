"""DivProbRanker (mirror of ptranking/ltr_diversification/score_and_sort/div_prob_ranker.py and base/div_mdn_ranker.py).

The scorer (pointsf or listsf, both over [q, d, q*d]) outputs 2 values per document for K = 1 and 3K for a K-component
mixture; a Gaussian head turns them into a mean and a variance per document.  One fused kernel per batch applies the
head, computes the loss over the pairwise probabilities P(j above i) = erfc((mu_i - mu_j) / sqrt(2 (v_i + v_j))) / 2 and
returns its gradient w.r.t. the raw output (ptrb200_divprob_fwd_bwd); the reference builds [1, n, n] and [m, n, n]
temporaries per query and differentiates them with autograd.  With the reference's one query per step the two agree;
``queries_per_step`` > 1 sums the queries' losses.  Evaluation sorts by the kernel's sort key (ptrb200_divprob_sort_key).
"""
from ..base.diversity_ranker import DiversityNeuralRanker
from ... import ops

SRD_METRIC = ['aNDCG', 'nERR-IA']
SORT_ID = ['ExpRele', 'RERAR', 'RiskAware']


def check_divprob_config(sf_para_dict, model_para_dict):
    """Refuse the configurations this class does not build, before any device is touched."""
    opt_id = model_para_dict['opt_id']
    assert opt_id in ['PairCLS', 'LambdaPairCLS', 'SuperSoft', 'Portfolio']
    if 'Portfolio' == opt_id:
        raise NotImplementedError("DivProbRanker opt_id='Portfolio' is not built: it needs cvxpy / cvxpylayers, and the "
                                  "reference hard-codes its portfolio problem to 50 assets")
    if model_para_dict['cluster']:
        raise NotImplementedError("DivProbRanker cluster=True is not built: it trains K separate scorers, and the "
                                  "reference concatenates their outputs along the document axis before its view")
    if sf_para_dict['sf_id'] not in ('pointsf', 'listsf'):
        raise NotImplementedError(f"DivProbRanker sf_id={sf_para_dict['sf_id']!r} is not built (pointsf and listsf "
                                  f"are; listsf_co's correlated variances are out of scope)")
    if opt_id in ('SuperSoft', 'LambdaPairCLS') and not model_para_dict['opt_ideal']:
        raise NotImplementedError("DivProbRanker opt_ideal=False is not built: the reference's SuperSoft-aNDCG branch "
                                  "then gathers a [1, 1, n] slice instead of resorting P, its nERR-IA branch returns a "
                                  "tuple, and its parameter grid never sets it")
    assert model_para_dict['K'] >= 1
    assert model_para_dict['sort_id'] in SORT_ID
    if 'SuperSoft' == opt_id:
        assert model_para_dict['metric'] in SRD_METRIC


class DivProbRanker(DiversityNeuralRanker):
    """A family of diversified ranking methods based on Mixture Density Networks (div_prob_ranker.py:234-359).  The
    checkpoint keys are the reference's: the pointsf state_dict, or {'encoder', 'uni_sf'} for listsf."""

    def __init__(self, sf_para_dict=None, model_para_dict=None, gpu=False, device=None):
        check_divprob_config(sf_para_dict, model_para_dict)
        self.K, self.cluster = model_para_dict['K'], model_para_dict['cluster']
        self.sort_id, self.limit_delta = model_para_dict['sort_id'], model_para_dict['limit_delta']
        self.b = 0.1
        # mean and raw variance, or mixing logit, mean and raw variance per component (div_mdn_ranker.py:48-56), set in
        # the caller's dict as the reference does
        sf_para_dict[sf_para_dict['sf_id']]['out_dim'] = 2 if 1 == self.K else 3 * self.K
        self.out_dim = sf_para_dict[sf_para_dict['sf_id']]['out_dim']
        super().__init__(id='DivProbRanker', sf_para_dict=sf_para_dict, gpu=gpu, device=device)
        self.stop_check_freq = 10
        self.opt_id = model_para_dict['opt_id']
        self.beta = 0.5  # i.e., alpha in alpha-nDCG
        self.opt_ideal, self.norm, self.top_k, self.metric = True, False, None, None
        if 'LambdaPairCLS' == self.opt_id:
            self.opt_ideal = model_para_dict['opt_ideal']
            self.norm = model_para_dict['norm']
        elif 'SuperSoft' == self.opt_id:
            self.opt_ideal = model_para_dict['opt_ideal']
            self.top_k = model_para_dict['top_k']
            self.metric = model_para_dict['metric']

    # ---- hooks of DiversityNeuralRanker ------------------------------------------------------------------------- #
    def split_list_order(self):
        """Both scorers read [q, d, q*d] (DivMDNRanker.div_switch_forward, div_mdn_ranker.py:212-220)."""
        return True

    def split_sort_keys(self, preds, sp):
        return ops.divprob_sort_key(preds.view(-1, self.out_dim), self.sort_id, K=self.K, limit_delta=self.limit_delta,
                                    offsets=sp.offsets, max_len=sp.max_len)

    # ---- scorer output ------------------------------------------------------------------------------------------ #
    def _raw(self, q_repr, doc_reprs):
        """One query: q_repr [1,F], doc_reprs [n,F] -> raw scorer output [n, out_dim]."""
        n = doc_reprs.size(0)
        if 'listsf' == self.sf_id:
            return self.list_div_forward(q_repr, doc_reprs).view(n, self.out_dim)
        X = ops.div_list_features(q_repr.reshape(1, -1), doc_reprs.reshape(1, n, -1))
        return self.point_sf(X).view(n, self.out_dim)

    def div_forward(self, q_repr, doc_reprs):
        """div_mdn_ranker.py:248-299 -> (mus, vars), each [1, n]."""
        mu, var = ops.divprob_head(self._raw(q_repr, doc_reprs), K=self.K, limit_delta=self.limit_delta)
        return mu.view(1, -1), var.view(1, -1)

    def div_predict(self, q_repr, doc_reprs):
        """div_mdn_ranker.py:301-326: mu (ExpRele), 1 / expected rank (RERAR) or mu - 0.1 var (RiskAware), [1, n]."""
        raw = self._raw(q_repr, doc_reprs)
        return ops.divprob_sort_key(raw.unsqueeze(0), self.sort_id, K=self.K, limit_delta=self.limit_delta)

    # ---- training ----------------------------------------------------------------------------------------------- #
    def div_train(self, train_data, epoch_k=None, queries_per_step=None):
        """DiversityNeuralRanker.div_train without the stop check: DivMDNRanker.div_train_op never asks to stop."""
        return super().div_train(train_data, epoch_k=None, queries_per_step=queries_per_step)

    def div_train_op(self, q_repr, doc_reprs, q_doc_rele_mat, **kwargs):
        """div_mdn_ranker.py:329-337: one query's step from host or device tensors; never asks to stop."""
        raw = self._raw(q_repr.to(self.device), doc_reprs.to(self.device))
        rele = ops.SubtopicRele.pack([q_doc_rele_mat], self.device)
        kwargs.pop('epoch_k', None)
        return self.div_custom_loss_function(raw.view(1, -1), rele, **kwargs), False

    def div_custom_loss_function(self, batch_preds, q_doc_rele_mat, **kwargs):
        """div_prob_ranker.py:295-359 with the Gaussian head fused in.  ``batch_preds``: the raw scorer output, [1, n *
        out_dim] for one query or flat [total * out_dim] with ``offsets``/``max_len``; ``q_doc_rele_mat``: the batch's
        ops.SubtopicRele."""
        assert 'presort' in kwargs and kwargs['presort'] is True
        offsets = kwargs.get('offsets')
        raw = batch_preds.view(-1, self.out_dim) if offsets is not None else batch_preds.view(1, -1, self.out_dim)
        batch_loss, _ = ops.divprob_loss(raw, q_doc_rele_mat, opt_id=self.opt_id, metric=self.metric, K=self.K,
                                         limit_delta=self.limit_delta, top_k=self.top_k, norm=self.norm,
                                         offsets=offsets, max_len=kwargs.get('max_len'))
        self.backward_and_step(batch_loss)
        return batch_loss

    def uniform_eval_setting(self, **kwargs):
        """div_prob_ranker.py:289-293: SuperSoft validates on the metric it optimises."""
        eval_dict = kwargs['eval_dict']
        if 'SuperSoft' == self.opt_id and eval_dict["do_validation"] and not eval_dict['vali_metric'] == self.metric:
            eval_dict['vali_metric'] = self.metric
