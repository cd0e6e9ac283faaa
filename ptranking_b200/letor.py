"""LETOR text files read on the device: ``read_letor`` -> :class:`LetorSplit`, and the ``LTRDataset`` drop-in.

The reference reads each split with ``LTRDataset`` (ptranking/data/data_utils.py:553-647): the text is parsed a line at a
time with ``str.split`` and ``float()``, documents are collected per qid, each query is scaled with an sklearn scaler,
labels are clipped, small queries dropped and documents presorted.  Here the host reads the file into pinned memory
and copies the bytes to the device once; every later step runs in the kernels of csrc/letor.cu (DESIGN.md "Reading
LETOR files on the device").  Only sizes, the undecided-token list and the kept qid strings come back to the host.

    split = read_letor("Fold1/train.txt", data_dict, presort=True, seed=0)
    batches = RaggedBatches.from_split(split, docs_per_batch=1 << 18)

Values match the reference's: labels and features are Python ``float()`` of each token (exactly, see
letor_float.cuh); unscaled rows are bit-equal, scaled rows are the float64 scalers rounded once to fp32.  The one
kept difference is tie order under ``presort``, random in both (here from a seeded device stream).
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch
import torch.utils.data as tud

from . import _lib

MSLETOR_LIST = ("MQ2007_List", "MQ2008_List")
YAHOO_LTR = ("Set1", "Set2")                       # zero-indexed feature ids (data_utils.py:495-496)
ISTELLA_LTR = ("Istella_S", "Istella", "Istella_X")
_HAS_COMMENT = {"MQ2007_Super": True, "MQ2008_Super": True, "MQ2007_Semi": True, "MQ2008_Semi": True,
                "MQ2007_List": True, "MQ2008_List": True, "IRGAN_MQ2008_Semi": True, "MSLRWEB10K": False,
                "MSLRWEB30K": False, "Set1": False, "Set2": False, "5FoldSet1": False, "5FoldSet2": False,
                "Istella_S": False, "Istella": False, "Istella_X": True}
_SCALERS = {None: 0, "StandardScaler": 1, "MinMaxScaler": 2}        # PTRB200_LETOR_*
_UNDECIDED_CAP = 4096


@dataclass
class LetorSplit:
    """One split on the device: ``X [total, W]`` (fp32 or bf16), ``y [total]`` fp32, ``offsets [B+1]`` int32 (query b owns
    rows offsets[b]:offsets[b+1]), the same offsets on the host, the qid strings in order of first appearance, the
    longest query, and how many tokens were handed to Python's float() (0 on ordinary files)."""
    X: torch.Tensor
    y: torch.Tensor
    offsets: torch.Tensor
    offsets_host: np.ndarray
    qids: List[str]
    max_len: int
    host_tokens: int = 0

    @property
    def num_features(self) -> int:
        return int(self.X.shape[1])

    def __len__(self) -> int:
        return len(self.qids)

    def query(self, b: int):
        a, e = int(self.offsets_host[b]), int(self.offsets_host[b + 1])
        return self.qids[b], self.X[a:e], self.y[a:e]


def _check_config(data_dict: dict, feature_dtype: torch.dtype) -> None:
    """Refuse what is not built, before any device work."""
    if feature_dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"feature_dtype must be torch.float32 or torch.bfloat16, got {feature_dtype}")
    if data_dict.get("scale_data"):
        sid = data_dict.get("scaler_id")
        if sid in ("RobustScaler", "SLog1P"):
            raise NotImplementedError(f"scaler_id={sid!r}: the per-query median/IQR and symmetric-log scalers are not "
                                      "built on the device; use StandardScaler, MinMaxScaler or no scaling")
        if sid not in _SCALERS or sid is None:
            raise ValueError(f"unknown scaler_id {sid!r}")
        if data_dict.get("scaler_level", "QUERY") == "DATASET":
            raise NotImplementedError("scaler_level='DATASET': only per-query scaling is built on the device")


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _check(rc, what):
    _lib.check(rc, what)


def _host_floats(host: np.ndarray, entries: np.ndarray):
    """float() of the undecided tokens: (byte offset, length, destination) rows -> (destinations, values).  A feature id
    repeated on one line can list one destination twice: the token further right wins, as on the device."""
    last = {}
    for o, n, d in sorted(entries.tolist()):
        last[d] = (o, n)
    dst = np.fromiter(last.keys(), dtype=np.int64, count=len(last))
    vals = [float(host[o:o + n].tobytes().decode("iso-8859-1")) for o, n in last.values()]
    return dst, np.asarray(vals, dtype=np.float64)


def read_letor(file: str, data_dict: dict, presort: bool, seed: int = 0, feature_dtype: torch.dtype = torch.float32,
               device=None) -> LetorSplit:
    """Read one LETOR split file into a device :class:`LetorSplit` with the reference's semantics
    (data_utils.py:420-549).  ``data_dict`` keys are the reference's: data_id, scale_data, scaler_id, scaler_level,
    binary_rele, unknown_as_zero, min_docs, min_rele (has_comment is taken from data_id when absent).  ``seed`` drives
    the tie shuffle of ``presort``; ``feature_dtype`` torch.bfloat16 rounds the fp32 rows to bf16 (nearest even)."""
    _check_config(data_dict, feature_dtype)
    data_id = data_dict["data_id"]
    has_comment = bool(data_dict.get("has_comment", _HAS_COMMENT.get(data_id, False)))
    one_indexed = not (data_id in YAHOO_LTR and not has_comment)
    scale = bool(data_dict.get("scale_data"))
    cfg = _lib.LetorCfg(scaler=_SCALERS[data_dict.get("scaler_id")] if scale else 0,
                   clip_istella=int(scale and data_id in ISTELLA_LTR), rank_labels=int(data_id in MSLETOR_LIST),
                   binary_rele=int(bool(data_dict.get("binary_rele"))), unknown_as_zero=int(bool(data_dict.get("unknown_as_zero"))),
                   min_docs=int(data_dict.get("min_docs") or 0), min_rele=int(data_dict.get("min_rele") or 0),
                   seed=int(seed) & (2 ** 64 - 1))
    lib = _lib.load()
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    nbytes = os.path.getsize(file)
    if nbytes == 0:
        raise _lib.B200LibraryError(f"{file}: empty file")
    with torch.cuda.device(dev):
        host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        hv = host.numpy()
        with open(file, "rb") as f:
            if f.readinto(memoryview(hv)) != nbytes:
                raise OSError(f"{file}: short read")
        text = host.to(dev, non_blocking=True)
        st = _stream()
        ws = torch.empty(int(lib.ptrb200_letor_index_workspace_bytes(nbytes)), dtype=torch.uint8, device=dev)
        n_lines = C.c_int64()
        _check(lib.ptrb200_letor_count_lines(text.data_ptr(), nbytes, ws.data_ptr(), C.byref(n_lines), st), "letor_count_lines")
        L = int(n_lines.value)
        line_start = torch.empty(L + 1, dtype=torch.int64, device=dev)
        _check(lib.ptrb200_letor_index_lines(text.data_ptr(), nbytes, ws.data_ptr(), L, line_start.data_ptr(), st), "letor_index_lines")
        del ws
        labels = torch.empty(L, dtype=torch.float64, device=dev)
        span = torch.empty(2 * L, dtype=torch.int64, device=dev)
        info = torch.empty(3, dtype=torch.int64, device=dev)
        info_h = (C.c_ulonglong * 3)()
        host_tokens = 0

        def parse(X, W):
            cap = _UNDECIDED_CAP
            while True:
                und = torch.empty(3 * cap, dtype=torch.int64, device=dev)
                _check(lib.ptrb200_letor_parse(text.data_ptr(), line_start.data_ptr(), L, int(one_indexed), int(has_comment),
                                               labels.data_ptr(), span.data_ptr(), None if X is None else X.data_ptr(), W,
                                               und.data_ptr(), cap, info.data_ptr(), info_h, st), f"letor_parse({file})")
                if int(info_h[2]) <= cap:
                    return int(info_h[0]), und[: 3 * int(info_h[2])].view(-1, 3).cpu().numpy()
                cap = int(info_h[2])

        W, und = parse(None, 0)
        if len(und):
            dst, vals = _host_floats(hv, und)
            labels[torch.from_numpy(-1 - dst).to(dev)] = torch.from_numpy(vals).to(dev)
            host_tokens += len(und)
        X64 = torch.empty((L, W), dtype=torch.float64, device=dev)
        _, und = parse(X64, W)
        if len(und):
            dst, vals = _host_floats(hv, und)
            X64.view(-1)[torch.from_numpy(dst).to(dev)] = torch.from_numpy(vals).to(dev)
            host_tokens += len(und)

        gws = torch.empty(int(lib.ptrb200_letor_group_workspace_bytes(L)), dtype=torch.uint8, device=dev)
        stats = (C.c_int * 3)()
        lines = torch.empty(L, dtype=torch.int32, device=dev)
        _check(lib.ptrb200_letor_group(text.data_ptr(), span.data_ptr(), L, gws.data_ptr(), lines.data_ptr(), None, None, 0,
                                       stats, st), "letor_group")
        B = int(stats[0])
        offsets = torch.empty(B + 1, dtype=torch.int32, device=dev)
        counts = torch.empty(B, dtype=torch.int32, device=dev)
        _check(lib.ptrb200_letor_group(text.data_ptr(), span.data_ptr(), L, gws.data_ptr(), lines.data_ptr(),
                                       offsets.data_ptr(), counts.data_ptr(), B, stats, st), f"letor_group({file})")
        max_len = int(stats[1])
        del gws, counts

        y_grouped = torch.empty(L, dtype=torch.float32, device=dev)
        kept_docs = torch.empty(B, dtype=torch.int32, device=dev)
        kept = torch.empty(B, dtype=torch.int32, device=dev)
        out_base = torch.empty(B, dtype=torch.int32, device=dev)
        order = torch.empty(L, dtype=torch.int32, device=dev) if presort else None
        scan_tmp = torch.empty(2 + 2 * ((B + 4095) // 4096), dtype=torch.int32, device=dev)
        sel = (C.c_int * 2)()
        _check(lib.ptrb200_letor_select(labels.data_ptr(), lines.data_ptr(), offsets.data_ptr(), B, max_len, C.byref(cfg),
                                        y_grouped.data_ptr(), kept_docs.data_ptr(), kept.data_ptr(), out_base.data_ptr(),
                                        None if order is None else order.data_ptr(), scan_tmp.data_ptr(), sel, st), "letor_select")
        total, K = int(sel[0]), int(sel[1])
        X = torch.empty((total, W), dtype=feature_dtype, device=dev)
        y = torch.empty(total, dtype=torch.float32, device=dev)
        out_offsets = torch.zeros(K + 1, dtype=torch.int32, device=dev)
        if K:
            _check(lib.ptrb200_letor_gather(X64.data_ptr(), W, lines.data_ptr(), offsets.data_ptr(), B, kept_docs.data_ptr(),
                                            kept.data_ptr(), out_base.data_ptr(), None if order is None else order.data_ptr(),
                                            y_grouped.data_ptr(), C.byref(cfg), X.data_ptr(),
                                            _lib.DTYPE_BF16 if feature_dtype == torch.bfloat16 else _lib.DTYPE_F32,
                                            y.data_ptr(), out_offsets.data_ptr(), st), "letor_gather")
        # qid strings of the kept queries: the first line of each query holds its qid bytes
        keep = kept_docs > 0
        first = lines[offsets[:-1].long()][keep].long()
        sp = span.view(-1, 2)[first].cpu().numpy()
        qids = [hv[o:o + n].tobytes().decode("iso-8859-1") for o, n in sp]
        offsets_host = out_offsets.cpu().numpy().astype(np.int64)
    lens = np.diff(offsets_host)
    return LetorSplit(X=X, y=y, offsets=out_offsets, offsets_host=offsets_host, qids=qids,
                      max_len=int(lens.max()) if len(lens) else 0, host_tokens=host_tokens)


def _default_data_dict(data_id: str) -> dict:
    """LTRDataset.get_default_data_dict (data_utils.py:650-666) for the keys read_letor uses."""
    scaled = data_id in ("MSLRWEB10K", "MSLRWEB30K") or data_id in ISTELLA_LTR
    return dict(data_id=data_id, min_docs=1, min_rele=1, binary_rele=False, unknown_as_zero=False,
                scale_data=scaled, scaler_id="StandardScaler" if scaled else None, scaler_level="QUERY" if scaled else None,
                has_comment=_HAS_COMMENT[data_id])


class LTRDataset(tud.Dataset):
    """Drop-in for the reference's ``LTRDataset`` (data_utils.py:553-673) backed by a device :class:`LetorSplit`.

    ``list_torch_Qs``, ``__len__`` and ``__getitem__`` give ``(qid, X[n, W], y[n])`` as views into the split's device
    tensors, so the reference's ``LETORSampler`` and ``DataLoader`` work unchanged and ``NeuralRanker.train``'s upload
    is a no-op copy.  ``buffer`` is accepted for the constructor's sake and writes no pickle: re-reading a file on the
    device costs less than loading the reference's buffers.  ``hot`` and label masking are not built."""

    def __init__(self, split_type, file, data_id=None, data_dict=None, eval_dict=None, presort=False, hot=False, buffer=True,
                 seed: int = 0, feature_dtype: torch.dtype = torch.float32):
        assert data_id is not None or data_dict is not None
        if hot:
            raise NotImplementedError("hot=True (one-hot labels and per-grade counts) is not built on the device")
        if eval_dict is not None and eval_dict.get("mask_label"):
            raise NotImplementedError("mask_label: label masking is not built on the device")
        if data_dict is None:
            data_dict = _default_data_dict(data_id)
        self.hot, self.presort, self.split_type = hot, presort, split_type
        self.label_type = data_dict.get("label_type")
        self.data_id = data_dict["data_id"]
        self.split = read_letor(file, data_dict, presort=presort, seed=seed, feature_dtype=feature_dtype)
        self.list_torch_Qs = [self.split.query(b) for b in range(len(self.split))]

    def __len__(self):
        return len(self.list_torch_Qs)

    def __getitem__(self, index):
        return self.list_torch_Qs[index]
