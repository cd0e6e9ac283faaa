"""Parameter containers of the stacked feed-forward scorer.

Mirror of ``get_stacked_FFNet`` (ptranking/base/utils.py:288-356): identical module
names, hence identical ``state_dict`` keys (``ff_2.weight``, ``bn_2.bn.weight``,
``bn_2.gamma`` ...), identical xavier-normal initialisation -- but ``forward`` hands the
whole stack to the fused CUDA kernels (ptranking_b200/csrc/ffnet.cu) instead of running
nn.Sequential through ATen.
"""
from __future__ import annotations

import os

import torch
import torch.nn as nn

from .. import ops

SUPPORTED_AF = ("R", "GE", "S", "T", "CE", "E", "LR", "SE")


class _BNParams(nn.Module):
    """Holder with the key layout of LTRBatchNorm (base/utils.py:201-223): ``.bn.weight/.bn.bias``."""

    def __init__(self, width, affine):
        super().__init__()
        self.bn = nn.BatchNorm1d(width, momentum=0.1, affine=affine, track_running_stats=False)


class _BN2Params(nn.Module):
    """Holder with the key layout of LTRBatchNorm2 (base/utils.py:249-282)."""

    def __init__(self, width, affine, device=None):
        super().__init__()
        shape = (1, 1, width)
        self.gamma = nn.Parameter(torch.ones(shape, device=device))
        self.beta = nn.Parameter(torch.zeros(shape, device=device))
        self.affine = affine
        if affine:
            self.weight = nn.Parameter(torch.ones(shape, device=device))
            self.bias = nn.Parameter(torch.zeros(shape, device=device))


class StackedFFNet(nn.Module):
    """Dropout -> Linear -> (BN|BN2) -> AF per hidden layer, Linear [-> norm -> TL_AF] tail."""

    def __init__(self, ff_dims, AF=None, TL_AF=None, apply_tl_af=False, dropout=0.1,
                 BN=True, bn_type=None, bn_affine=False, device=None, math_mode=None, bn_per_query=False,
                 pad_output=False):
        """``bn_per_query`` (bn_type 'BN' only): normalise each query over its own documents, as the reference's BN does
        when it scores one query per call (the diversification rankers).  The parameters and checkpoint keys stay
        LTRBatchNorm's; the kernels run BN2's per-query statistics with gamma/beta = bn.weight/bn.bias (constant 1 / 0
        without affine) and no second affine.
        ``pad_output``: the tensor-core kernels take output widths up to 4 or multiples of 4, and per-query statistics
        over a ragged batch run on them only; any other width sends the whole net to the fp32 SIMT kernels, which refuse
        ragged per-query batches.  With ``pad_output`` such an output layer (DivProbRanker's 3K mixture outputs) is
        computed zero-padded to the next multiple of 4 -- zero weight rows and bias, and for a normalised output layer
        scale 1 / shift 0 -- and the first ff_dims[-1] columns are returned.  The padded columns are constant 0 before
        the norm, so they change neither the other columns' statistics nor their gradients; parameters and checkpoint
        keys keep their own shapes."""
        super().__init__()
        # "3xtf32" (default): wgmma tensor cores with the fp32-equivalent 3-pass TF32 split;
        # "tf32": single pass; "simt": fp32 FMA kernels (also the fallback for widths the MMA tiles reject)
        math_mode = math_mode or os.environ.get("PTRANKING_B200_MATH", "3xtf32")
        assert ff_dims is not None and len(ff_dims) >= 2
        for code in ([AF] if len(ff_dims) > 2 else []) + ([TL_AF] if apply_tl_af else []):
            if code not in SUPPORTED_AF:
                raise NotImplementedError(f"activation {code!r}")     # get_AF's broken / unsupported branches
        if BN and bn_type not in ("BN", "BN2"):
            raise NotImplementedError(bn_type)
        if bn_per_query and not (BN and bn_type == "BN"):
            raise ValueError("bn_per_query applies to bn_type='BN' only")
        L = len(ff_dims)
        self._const_grads = []      # gradient sinks of the constant gamma/beta of a non-affine per-query BN
        # parameter tensors in the order the C ABI expects them; (module, buffer) names stand for those constants, which
        # .to() replaces
        self._order = []
        for i in range(1, L):
            self._last = len(self._order)       # where the output layer's tensors begin, after the loop
            lin = nn.Linear(ff_dims[i - 1], ff_dims[i])
            nn.init.xavier_normal_(lin.weight)
            self.add_module(f"ff_{i + 1}", lin)
            self._order += [lin.weight, lin.bias]
            has_act = i < L - 1 or apply_tl_af
            if has_act and BN:
                if bn_type == "BN":
                    holder = _BNParams(ff_dims[i], bn_affine)
                    if bn_affine:
                        self._order += [holder.bn.weight, holder.bn.bias]
                    elif bn_per_query:
                        holder.register_buffer("unit_gamma", torch.ones(ff_dims[i]), persistent=False)
                        holder.register_buffer("zero_beta", torch.zeros(ff_dims[i]), persistent=False)
                        self._order += [(f"bn_{i + 1}", "unit_gamma"), (f"bn_{i + 1}", "zero_beta")]
                else:
                    holder = _BN2Params(ff_dims[i], bn_affine, device=device)
                    self._order += [holder.gamma, holder.beta]
                    if bn_affine:
                        self._order += [holder.weight, holder.bias]
                self.add_module(f"bn_{i + 1}", holder)
        self.bn_per_query = bool(bn_per_query)
        norm = ("BN2" if bn_per_query else bn_type) if BN else None
        out = ff_dims[-1]
        self._pad_out = (-out) % 4 if pad_output and out > 4 else 0
        self.spec = ops.FFNetSpec(list(ff_dims[:-1]) + [out + self._pad_out], AF if L > 2 else None,
                                  TL_AF if apply_tl_af else None, norm, bn_affine and not bn_per_query, dropout,
                                  math_mode=math_mode)

    def ordered_parameters(self):
        ps = [getattr(getattr(self, e[0]), e[1]) if isinstance(e, tuple) else e for e in self._order]
        if self._pad_out:
            # the output layer: weight and bias with zero rows appended, then its norm's (scale, shift) pairs -- gamma
            # and beta, and BN2's affine weight and bias -- with 1 / 0
            k = self._last
            w = ps[k]
            ps[k] = torch.cat((w, w.new_zeros(self._pad_out, w.shape[1])))
            for j in range(k + 1, len(ps)):
                t = ps[j]
                fill = t.new_ones(self._pad_out) if (j - k) % 2 == 0 else t.new_zeros(self._pad_out)
                ps[j] = torch.cat((t, fill))
        return ps

    def _grad_targets(self):
        """p.grad of every parameter, and a scratch sink for each constant -- or None while some gradient storage is
        missing."""
        targets = []
        consts = 0
        for p in self.ordered_parameters():
            if isinstance(p, nn.Parameter):
                if p.grad is None or not p.grad.is_contiguous():
                    return None
                targets.append(p.grad)
            else:
                if consts == len(self._const_grads) or self._const_grads[consts].shape != p.shape \
                        or self._const_grads[consts].device != p.device:
                    self._const_grads[consts:consts + 1] = [torch.empty_like(p)]
                targets.append(self._const_grads[consts])
                consts += 1
        return targets

    def forward(self, X, offsets=None, max_len=None):
        """[B,n,F] (or [rows,F]) -> [B,n,out].  ``offsets``/``max_len`` describe a ragged batch ([total_docs,F] rows cut
        into queries): batch-level BN and norm-free nets see one long list; per-query BN2 needs the query boundaries."""
        ragged_bn2 = offsets is not None and self.spec.norm == "BN2"       # per-query statistics need the boundaries
        squeeze = X.dim() == 2 and not ragged_bn2
        if squeeze:
            X = X.unsqueeze(0)
        # when every parameter already owns gradient storage (the ranker's flat bucket), the backward kernels write
        # into it directly instead of handing autograd 2 tensors per layer to accumulate
        targets = None
        if torch.is_grad_enabled() and getattr(self, "write_through_grads", False) and not self._pad_out:
            targets = self._grad_targets()
        if ragged_bn2:
            if X.dim() != 2:
                raise ValueError("a ragged batch is [total_docs, F]")
            out = ops.ffnet_apply(X, self.spec, self.ordered_parameters(), training=self.training, grad_targets=targets,
                                  offsets=offsets, max_len=max_len)
            return out[:, :out.shape[1] - self._pad_out].contiguous() if self._pad_out else out
        out = ops.ffnet_apply(X, self.spec, self.ordered_parameters(), training=self.training, grad_targets=targets)
        if self._pad_out:
            out = out[..., :out.shape[-1] - self._pad_out].contiguous()
        return out.squeeze(0) if squeeze else out


def get_stacked_FFNet(ff_dims=None, AF=None, TL_AF=None, apply_tl_af=False, dropout=0.1,
                      BN=True, bn_type=None, bn_affine=False, device='cpu', split_penultimate_layer=False):
    """Same call signature as the reference factory (base/utils.py:288)."""
    if split_penultimate_layer:
        raise NotImplementedError("split_penultimate_layer is only used by out-of-scope models")
    return StackedFFNet(ff_dims, AF=AF, TL_AF=TL_AF, apply_tl_af=apply_tl_af, dropout=dropout,
                        BN=BN, bn_type=bn_type, bn_affine=bn_affine, device=device)
