"""NeuralRanker / Evaluator with the reference's method set (ptranking/base/ranker.py:28-65,
:67-95, :189-200, :479-630) driving the CUDA kernels.

Differences kept deliberately small and listed in DESIGN.md: tensors live on the CUDA
device for the whole step; nDCG is computed by the in-CTA sort kernel on the device
(the reference copies predictions to the host and sorts there, ranker.py:46-50)."""
from __future__ import annotations

from enum import Enum, auto, unique

import torch
import torch.optim as optim
from torch.optim.lr_scheduler import StepLR

from .. import ops
from .. import dist as b200dist


class FlatAdam(optim.Optimizer):
    """torch.optim.Adam as the reference configures it (ranker.py:512-525: lr, weight_decay, PyTorch defaults otherwise) run
    as ONE kernel over the flat parameter / gradient buffers of a :class:`dist.GradBucket` (ops.adam_step).  It is a
    torch Optimizer, so StepLR (ranker.py:525) drives ``param_groups[0]['lr']`` as usual."""

    def __init__(self, params, bucket, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self.bucket = bucket
        self.exp_avg = torch.zeros_like(bucket.flat_param)
        self.exp_avg_sq = torch.zeros_like(bucket.flat_param)
        self.num_steps = 0

    @torch.no_grad()
    def step(self, closure=None):
        if not self.bucket.params_are_flat():
            raise RuntimeError("FlatAdam: a parameter was re-allocated outside the flat buffer (use copy_ / load_state_dict)")
        g = self.param_groups[0]
        self.num_steps += 1
        ops.adam_step(self.bucket.flat_param, self.bucket.flat, self.exp_avg, self.exp_avg_sq, self.num_steps,
                      lr=g['lr'], betas=g['betas'], eps=g['eps'], weight_decay=g['weight_decay'], peer=self.bucket.peer_group())
        self.bucket.advance()


class FlatAdagrad(optim.Optimizer):
    """torch.optim.Adagrad(lr, weight_decay) -- the list scorer's default (parameter.py:157-162) -- as one kernel."""

    def __init__(self, params, bucket, lr=1e-2, lr_decay=0.0, eps=1e-10, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, lr_decay=lr_decay, eps=eps, weight_decay=weight_decay))
        self.bucket = bucket
        self.state_sum = torch.zeros_like(bucket.flat_param)
        self.num_steps = 0

    @torch.no_grad()
    def step(self, closure=None):
        if not self.bucket.params_are_flat():
            raise RuntimeError("FlatAdagrad: a parameter was re-allocated outside the flat buffer (use copy_ / load_state_dict)")
        g = self.param_groups[0]
        self.num_steps += 1
        ops.adagrad_step(self.bucket.flat_param, self.bucket.flat, self.state_sum, self.num_steps, lr=g['lr'],
                         lr_decay=g['lr_decay'], eps=g['eps'], weight_decay=g['weight_decay'], peer=self.bucket.peer_group())
        self.bucket.advance()


class FlatRMSprop(optim.Optimizer):
    """torch.optim.RMSprop(lr, weight_decay) (alpha=0.99, eps=1e-8, no momentum, not centered) as one kernel."""

    def __init__(self, params, bucket, lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, alpha=alpha, eps=eps, weight_decay=weight_decay))
        self.bucket = bucket
        self.square_avg = torch.zeros_like(bucket.flat_param)

    @torch.no_grad()
    def step(self, closure=None):
        if not self.bucket.params_are_flat():
            raise RuntimeError("FlatRMSprop: a parameter was re-allocated outside the flat buffer (use copy_ / load_state_dict)")
        g = self.param_groups[0]
        ops.rmsprop_step(self.bucket.flat_param, self.bucket.flat, self.square_avg, lr=g['lr'], alpha=g['alpha'],
                         eps=g['eps'], weight_decay=g['weight_decay'], peer=self.bucket.peer_group())
        self.bucket.advance()


@unique
class LABEL_TYPE(Enum):
    """Same members as ptranking.data.data_utils.LABEL_TYPE (data_utils.py:88-91)."""
    MultiLabel = auto()
    Permutation = auto()


def _is_multilabel(label_type) -> bool:
    return getattr(label_type, "name", label_type) == "MultiLabel"


class Evaluator:
    """nDCG evaluation API of ptranking.base.ranker.Evaluator."""

    def _scores_and_labels(self, batch_q_doc_vectors, batch_std_labels, offsets=None, max_len=None):
        dev = self.device
        # no autograd tape in evaluation: the scorer then runs forward-only (no backward by-products written, no
        # activation workspace kept alive).  The reference never disables grad here (ranker.py:623-630), which only
        # matters for its BN2 train/eval switch (SURVEY B4); these kernels use per-query statistics in both modes.
        with torch.no_grad():
            X = batch_q_doc_vectors.to(dev, non_blocking=True)
            preds = self.predict(X) if offsets is None else self.forward_ragged(X, offsets, max_len)
        return preds.detach(), batch_std_labels.to(dev, non_blocking=True)

    def _eval_batches(self, test_data, k=None):
        """-> (num_queries counted, preds, labels, ragged kwargs) per batch.  Dense batches are the reference's
        (ids, X[B,n,F], y[B,n]); ragged ones are data.RaggedBatches' (ids, X[total,F], y[total], offsets, max_len).
        With ``k`` given, lists shorter than k do not count (ranker.py:41-42 skips such batches; in a ragged batch the
        rule applies per query -- the kernel reports 0 for them)."""
        for batch in test_data:
            if len(batch) >= 5:
                ids, X, y, offsets, max_len = batch[:5]
                lens = (offsets[1:] - offsets[:-1]).cpu()
                counted = int((lens >= k).sum()) if k is not None else len(ids)
                if counted == 0:
                    continue
                off_d = offsets.to(self.device, non_blocking=True)
                preds, labels = self._scores_and_labels(X, y, off_d, max_len)
                yield counted, preds, labels, dict(offsets=off_d, max_len=max_len, buckets=batch[5] if len(batch) > 5 else None)
            else:
                ids, X, y = batch
                if k is not None and y.size(1) < k:
                    continue
                preds, labels = self._scores_and_labels(X, y)
                yield len(ids), preds, labels, {}

    def ndcg_at_k(self, test_data=None, k=10, label_type=LABEL_TYPE.MultiLabel, presort=False, device='cpu'):
        """ranker.py:31-65: average nDCG@k; batches with fewer than k documents are skipped (:41-42)."""
        assert _is_multilabel(label_type)
        self.eval_mode()
        num_queries = 0
        total = torch.zeros(1, device=self.device)
        for counted, preds, labels, rk in self._eval_batches(test_data, k=k):
            num_queries += counted
            total += ops.sum_f32(ops.ndcg_at_ks(preds, labels, [k], presort=presort, **rk))
        return (total / num_queries).cpu()

    def ndcg_at_ks(self, test_data=None, ks=[1, 5, 10], label_type=LABEL_TYPE.MultiLabel, presort=False, device='cpu'):
        """ranker.py:67-95."""
        assert _is_multilabel(label_type)
        self.eval_mode()
        num_queries = 0
        total = torch.zeros(len(ks), device=self.device)
        for counted, preds, labels, rk in self._eval_batches(test_data):
            total += ops.ndcg_at_ks(preds, labels, ks, presort=presort, **rk).sum(dim=0)
            num_queries += counted
        return (total / num_queries).cpu()

    def _metric_at_k(self, which, test_data, k, presort, max_label=None, skip_short=True):
        """shared body of nerr_at_k / ap_at_k / p_at_k (ranker.py:97-187): batches with fewer than k documents
        are skipped, the average runs over the remaining queries."""
        self.eval_mode()
        num_queries = 0
        total = torch.zeros(1, device=self.device)
        for counted, preds, labels, rk in self._eval_batches(test_data, k=k if skip_short else None):
            num_queries += counted
            vals = ops.adhoc_metrics_at_ks(preds, labels, [k], presort=presort, max_label=max_label, **rk)[which]
            total += ops.sum_f32(vals)
        return (total / num_queries).cpu()

    def nerr_at_k(self, test_data=None, k=10, label_type=LABEL_TYPE.MultiLabel, max_label=None, presort=False, device='cpu'):
        assert _is_multilabel(label_type)
        return self._metric_at_k(1, test_data, k, presort, max_label=max_label)

    def ap_at_k(self, test_data=None, k=10, presort=False, device='cpu'):
        return self._metric_at_k(2, test_data, k, presort)

    def p_at_k(self, test_data=None, k=10, device='cpu'):
        return self._metric_at_k(3, test_data, k, presort=False)

    def validation(self, vali_data=None, vali_metric=None, k=5, presort=False, max_label=None,
                   label_type=LABEL_TYPE.MultiLabel, device='cpu'):
        """ranker.py:189-200."""
        if 'nDCG' == vali_metric:
            return self.ndcg_at_k(test_data=vali_data, k=k, label_type=label_type, presort=presort, device=device)
        elif 'nERR' == vali_metric:
            return self.nerr_at_k(test_data=vali_data, k=k, label_type=label_type, max_label=max_label, presort=presort, device=device)
        elif 'AP' == vali_metric:
            return self.ap_at_k(test_data=vali_data, k=k, presort=presort, device=device)
        elif 'P' == vali_metric:
            return self.p_at_k(test_data=vali_data, k=k, device=device)
        else:
            raise NotImplementedError

    def adhoc_performance_at_ks(self, test_data=None, ks=[1, 5, 10], label_type=LABEL_TYPE.MultiLabel, max_label=None,
                                presort=False, device='cpu', need_per_q=False):
        """ranker.py:202-263: average nDCG / nERR / AP / P at every cutoff (one fused kernel per batch)."""
        assert _is_multilabel(label_type)
        self.eval_mode()
        num_queries = 0
        sums = [torch.zeros(len(ks), device=self.device) for _ in range(4)]
        per_q = [[] for _ in range(4)]
        for counted, preds, labels, rk in self._eval_batches(test_data):
            vals = ops.adhoc_metrics_at_ks(preds, labels, ks, presort=presort, max_label=max_label, **rk)
            for m in range(4):
                sums[m] += vals[m].sum(dim=0)
                if need_per_q:
                    per_q[m].append(vals[m].cpu())
            num_queries += counted
        avgs = [(s_ / num_queries).cpu() for s_ in sums]
        if need_per_q:
            return (*avgs, *per_q)
        return tuple(avgs)


class NeuralRanker(Evaluator):
    """ptranking/base/ranker.py:479-630."""

    def __init__(self, id='AbsRanker', sf_para_dict=None, weight_decay=1e-3, gpu=False, device=None):
        self.id = id
        self.gpu, self.device = gpu, device
        self.sf_para_dict = sf_para_dict
        self.sf_id = sf_para_dict['sf_id']
        self.opt, self.lr = sf_para_dict['opt'], sf_para_dict['lr']
        self.weight_decay = weight_decay
        self.stop_check_freq = 10
        self._require_cuda()

    def _require_cuda(self):
        if not self.gpu or self.device is None or not str(self.device).startswith('cuda'):
            raise RuntimeError("ptranking_b200 rankers run on a CUDA device only (gpu=True, device='cuda:N'); "
                               "there is no CPU fallback")

    def init(self):
        pass

    def get_parameters(self):
        pass

    def config_optimizer(self):
        """ranker.py:512-525: Adam | RMS | Adagrad with L2-in-gradient weight decay + StepLR(20, 0.5)."""
        params = list(self.get_parameters())
        self.grad_bucket = b200dist.GradBucket(params, align=4)     # one flat fp32 gradient buffer (one all-reduce per step)
        # every optimizer the reference offers is ONE fused kernel over the flat parameter / gradient / state buffers
        if self.opt not in ('Adam', 'RMS', 'Adagrad'):
            raise NotImplementedError
        self.grad_bucket.flatten_params()
        if 'Adam' == self.opt:      # the pointwise scorer's default
            self.optimizer = FlatAdam(params, self.grad_bucket, lr=self.lr, weight_decay=self.weight_decay)
        elif 'RMS' == self.opt:
            self.optimizer = FlatRMSprop(params, self.grad_bucket, lr=self.lr, weight_decay=self.weight_decay)
        else:                       # 'Adagrad': the list scorer's default (parameter.py:157-162)
            self.optimizer = FlatAdagrad(params, self.grad_bucket, lr=self.lr, weight_decay=self.weight_decay)
        self.scheduler = StepLR(self.optimizer, step_size=20, gamma=0.5)
        # data parallel: every replica must start from rank 0's weights (xavier_normal_ draws from the per-process
        # torch seed); the all-reduced gradient is only meaningful when applied to identical replicas
        b200dist.broadcast_parameters(self.grad_bucket, src=0)
        # ... and, on one node, the gradient sum moves into the optimizer kernel (NVLink peer memory; NCCL otherwise)
        self.grad_bucket.enable_peer()

    def backward_and_step(self, batch_loss):
        """The tail every reference loss class ends with (e.g. lambdarank.py:58-60), plus the
        data-parallel gradient all-reduce (sum: every reference loss is a sum over queries)."""
        self.grad_bucket.zero(skip_memset=getattr(self, 'grad_bucket_overwritten', False))
        if getattr(self, '_unit_grad', None) is None or self._unit_grad.device != batch_loss.device:
            self._unit_grad = torch.ones((), dtype=torch.float32, device=batch_loss.device)
        if getattr(self, 'grad_bucket_overwritten', False):
            self.grad_bucket.begin_overlap()               # layers' gradient slices go out as they complete
        batch_loss.backward(gradient=self._unit_grad)       # cached root gradient: no fill kernel per step
        self.grad_bucket.all_reduce()
        self.optimizer.step()

    def eval_mode(self):
        pass

    def train_mode(self):
        pass

    def save(self, dir, name):
        pass

    def load(self, file_model, **kwargs):
        pass

    def uniform_eval_setting(self, **kwargs):
        pass

    def stop_training(self, batch_preds):
        """ranker.py:547-561."""
        if torch.nonzero(batch_preds, as_tuple=False).size(0) <= 0:
            print('All zero error.\n')
            return True
        if torch.isnan(batch_preds).any():
            print('Including NaN error.')
            return True
        return False

    def train(self, train_data, epoch_k=None, **kwargs):
        """ranker.py:565-587, restructured for the device: the host->device copy of batch i+1 runs on a
        side stream while batch i trains (the reference copies synchronously from pageable memory, :577),
        and the blocking ``batch_loss.item()`` per batch (:584) becomes an asynchronous device->host copy
        of every step's loss into a pinned ring that is read once at the end."""
        self.train_mode()
        assert 'label_type' in kwargs and 'presort' in kwargs
        label_type, presort = kwargs['label_type'], kwargs['presort']
        num_queries = 0
        stop_training = False
        ring = self._loss_ring()
        host_sum, filled = 0.0, 0
        compute = torch.cuda.current_stream()
        copier = self._copy_stream()

        def upload(batch):
            # dense (ids, X[B,n,F], y[B,n]) as the reference's loaders yield, or ragged
            # (ids, X[total,F], y[total], offsets[B+1], max_len) from data.RaggedBatches
            ids, X, y = batch[0], batch[1], batch[2]
            with torch.cuda.stream(copier):
                Xd, yd = X.to(self.device, non_blocking=True), y.to(self.device, non_blocking=True)
                ragged = dict(offsets=batch[3].to(self.device, non_blocking=True), max_len=int(batch[4]),
                              buckets=batch[5] if len(batch) > 5 else None) if len(batch) >= 5 else {}
                ready = torch.cuda.Event()
                ready.record(copier)
            return ids, Xd, yd, ready, ragged

        it = iter(train_data)
        nxt = next(it, None)
        pending = upload(nxt) if nxt is not None else None
        while pending is not None:
            batch_ids, X, y, ready, ragged = pending
            nxt = next(it, None)
            pending = upload(nxt) if nxt is not None else None       # overlaps with the step below
            compute.wait_event(ready)
            X.record_stream(compute); y.record_stream(compute)
            if ragged:
                ragged['offsets'].record_stream(compute)
            num_queries += len(batch_ids)
            batch_loss, stop_training = self.train_op(X, y, batch_ids=batch_ids, epoch_k=epoch_k,
                                                      presort=presort, label_type=label_type, **ragged)
            if stop_training:
                break
            ring[filled].copy_(batch_loss.detach(), non_blocking=True)
            filled += 1
            if filled == ring.numel():
                compute.synchronize()
                host_sum += float(ring.double().sum())
                filled = 0
        compute.synchronize()
        host_sum += float(ring[:filled].double().sum())
        epoch_loss = torch.tensor([host_sum / max(num_queries, 1)], device=self.device)
        return epoch_loss, stop_training

    def _copy_stream(self):
        if getattr(self, '_copier', None) is None:
            self._copier = torch.cuda.Stream(device=self.device)
        return self._copier

    def _loss_ring(self):
        if getattr(self, '_ring', None) is None:
            self._ring = torch.zeros(1024, dtype=torch.float32).pin_memory()
        return self._ring

    def train_op(self, batch_q_doc_vectors, batch_std_labels, **kwargs):
        """ranker.py:589-603."""
        stop_training = False
        if kwargs.get('offsets') is not None:     # ragged batch: flat [total_docs, F] features, per-query offsets
            batch_preds = self.forward_ragged(batch_q_doc_vectors, kwargs['offsets'], kwargs['max_len'], buckets=kwargs.get('buckets'))
        else:
            batch_preds = self.forward(batch_q_doc_vectors)
        if 'epoch_k' in kwargs and kwargs['epoch_k'] is not None and kwargs['epoch_k'] % self.stop_check_freq == 0:
            stop_training = self.stop_training(batch_preds)
        return self.custom_loss_function(batch_preds, batch_std_labels, **kwargs), stop_training

    def custom_loss_function(self, batch_preds, batch_std_labels, **kwargs):
        pass

    def forward(self, batch_q_doc_vectors):
        pass

    def forward_ragged(self, flat_q_doc_vectors, offsets, max_len, buckets=None):
        """[total_docs, F] + int32 offsets[B+1] -> flat scores [total_docs] (no counterpart in the reference, whose
        batches are dense; SURVEY 8f-2).  ``buckets``: data.RaggedBatches' length classes [(q_begin, q_end, max_len)]."""
        raise NotImplementedError("this scorer has no ragged-batch path")

    def predict(self, batch_q_doc_vectors):
        """ranker.py:623-630."""
        return self.forward(batch_q_doc_vectors)

    @staticmethod
    def ragged_kwargs(kwargs):
        """The ragged-batch description a loss kernel needs, out of custom_loss_function's kwargs."""
        if kwargs.get('offsets') is None:
            return {}
        return dict(offsets=kwargs['offsets'], max_len=kwargs['max_len'], buckets=kwargs.get('buckets'))
