"""Host replica of the library's dropout mask stream (ptranking_b200/csrc/common.cuh), written from its specification.

Every dropout site regenerates its mask from a splitmix64 counter stream:

    key   = mix64(seed + GOLD * (index + 1))                 dropout_key(seed, index)
    draw  = mix64(key + GOLD * (elem >> 2))                  dropout_draw4(key, quad): 16 bits for each of 4 elements
    keep  = ((draw >> 16 * (elem & 3)) & 0xffff) >= thr      dropout_keep(key, elem, thr)
    thr   = (uint32)(float32(p) * 65536 + 0.5)               0 when p <= 0: dropout off
    scale = float32(65536) / float32(65536 - thr)            (not 1 / (1 - p): 1.11111867 against 1.11111111 at p = 0.1)

and the key index of a call is fixed by who draws it:

    stacked-FF net, offset o, Linear layer l:   o * 64 + l   element row * d_in(l) + col, row = b * n + i (dense) or
                                                             the flat document index (ragged); the last layer's input
                                                             has no dropout
    one-mask calls (elementwise dropout and     o * 64 + 63  elementwise: the flat index;
    attention), offset o                                     attention: (z * n + row) * n + col with z = b * H + h

The FF net uses at most PTRB200_MAX_FF_LAYERS (16) indices per offset, so the two domains never meet.  Everything here is
vectorised NumPy on uint64 (wrapping arithmetic, as in C): a mask over the 262144 x 136 bench batch is 9M draws.
"""
import numpy as np

GOLD = np.uint64(0x9E3779B97F4A7C15)
_M1 = np.uint64(0xBF58476D1CE4E5B9)
_M2 = np.uint64(0x94D049BB133111EB)
U64 = (1 << 64) - 1

FF_KEYS_PER_OFFSET = 64     # key indices an FF call at offset o owns: o*64 .. o*64+63
CALL_SLOT = 63              # the one-mask calls' slot inside an offset's block
MAX_FF_LAYERS = 16          # PTRB200_MAX_FF_LAYERS: an FF call uses slots 0 .. 14 at most


def _u64(x):
    if isinstance(x, (int, np.integer)):
        return np.uint64(int(x) & U64)
    return np.asarray(x, dtype=np.uint64)


def mix64(x):
    x = _u64(x)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(30))
        x = x * _M1
        x = x ^ (x >> np.uint64(27))
        x = x * _M2
        x = x ^ (x >> np.uint64(31))
    return x


def dropout_key(seed, index):
    with np.errstate(over="ignore"):
        return mix64(_u64(seed) + GOLD * (_u64(index) + np.uint64(1)))


def dropout_draw4(key, quad):
    with np.errstate(over="ignore"):
        return mix64(_u64(key) + GOLD * _u64(quad))


def keep(key, elem, thr):
    elem = _u64(elem)
    lane = (dropout_draw4(key, elem >> np.uint64(2)) >> (np.uint64(16) * (elem & np.uint64(3)))) & np.uint64(0xFFFF)
    return lane >= np.uint64(thr)


def threshold(p) -> int:
    p = np.float32(p)
    if not p > 0:
        return 0
    return int(np.uint32(p * np.float32(65536.0) + np.float32(0.5)))


def scale(p) -> np.float32:
    t = threshold(p)
    return np.float32(1.0) if t == 0 else np.float32(65536.0) / np.float32(65536 - t)


# ---- key rules of the callers ---------------------------------------------------------------------------------------
def ff_index(offset: int, layer: int) -> int:
    return offset * FF_KEYS_PER_OFFSET + layer


def call_index(offset: int) -> int:
    return offset * FF_KEYS_PER_OFFSET + CALL_SLOT


def ff_key(seed: int, offset: int, layer: int):
    return dropout_key(seed, ff_index(offset, layer))


def call_key(seed: int, offset: int):
    return dropout_key(seed, call_index(offset))


# ---- masks ----------------------------------------------------------------------------------------------------------
def keep_stream(key, count: int, thr: int) -> np.ndarray:
    """keep(key, e, thr) for e = 0 .. count-1 as a bool vector (one draw per 4 elements, lanes low bits first)."""
    quads = np.arange((count + 3) // 4, dtype=np.uint64)
    lanes = dropout_draw4(key, quads).astype("<u8").view("<u2")
    return lanes[:count] >= thr


def ff_mask(seed: int, offset: int, layer: int, p: float, rows: int, d_in: int) -> np.ndarray:
    """Keep mask [rows, d_in] of the input of Linear layer ``layer`` of an FF call (all True when p == 0)."""
    return keep_stream(ff_key(seed, offset, layer), rows * d_in, threshold(p)).reshape(rows, d_in)


def call_mask(seed: int, offset: int, p: float, shape) -> np.ndarray:
    """Keep mask of an elementwise dropout call over a tensor of ``shape`` (flat index), or of an attention call over
    its [B*H, n, n] probabilities."""
    count = int(np.prod(shape))
    return keep_stream(call_key(seed, offset), count, threshold(p)).reshape(shape)
