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
                 BN=True, bn_type=None, bn_affine=False, device=None, math_mode=None):
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
        L = len(ff_dims)
        self._order = []            # parameter tensors in the order the C ABI expects them
        for i in range(1, L):
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
                else:
                    holder = _BN2Params(ff_dims[i], bn_affine, device=device)
                    self._order += [holder.gamma, holder.beta]
                    if bn_affine:
                        self._order += [holder.weight, holder.bias]
                self.add_module(f"bn_{i + 1}", holder)
        self.spec = ops.FFNetSpec(ff_dims, AF if L > 2 else None, TL_AF if apply_tl_af else None,
                                  bn_type if BN else None, bn_affine, dropout, math_mode=math_mode)

    def ordered_parameters(self):
        return list(self._order)

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
        if torch.is_grad_enabled() and all(p.grad is not None and p.grad.is_contiguous() for p in self._order) \
                and getattr(self, "write_through_grads", False):
            targets = [p.grad for p in self._order]
        if ragged_bn2:
            if X.dim() != 2:
                raise ValueError("a ragged batch is [total_docs, F]")
            return ops.ffnet_apply(X, self.spec, self._order, training=self.training, grad_targets=targets,
                                   offsets=offsets, max_len=max_len)
        out = ops.ffnet_apply(X, self.spec, self._order, training=self.training, grad_targets=targets)
        return out.squeeze(0) if squeeze else out


def get_stacked_FFNet(ff_dims=None, AF=None, TL_AF=None, apply_tl_af=False, dropout=0.1,
                      BN=True, bn_type=None, bn_affine=False, device='cpu', split_penultimate_layer=False):
    """Same call signature as the reference factory (base/utils.py:288)."""
    if split_penultimate_layer:
        raise NotImplementedError("split_penultimate_layer is only used by out-of-scope models")
    return StackedFFNet(ff_dims, AF=AF, TL_AF=TL_AF, apply_tl_af=apply_tl_af, dropout=dropout,
                        BN=BN, bn_type=bn_type, bn_affine=bn_affine, device=device)
