"""A CPU restatement of the diversification list scorer (ltr_diversification/base/div_list_ranker.py:20-85) built from
oracle/ref_port.py's encoder layer, LayerNorm and stacked FF net, for the listsf parity tests; and the cases of the listsf
fixtures (tests/golden/make_golden_divlist.py) with their seeded starting weights and inputs, which are rebuilt here
rather than stored."""
import zlib

import numpy as np
import torch
import torch.nn as nn

from oracle import ref_port as rp

DEFAULT_LISTSF = dict(encoder_type='AttnDIN', n_heads=6, encoder_layers=6, ff_dims=[256, 128, 64], AF='R', TL_AF='GE',
                      apply_tl_af=False, BN=True, bn_type='BN', bn_affine=True)     # div_parameter.py:98-104
SMALL_LISTSF = dict(encoder_layers=2, ff_dims=[32, 16], AF='R', TL_AF='GE', apply_tl_af=False, BN=True, bn_type='BN',
                    bn_affine=True)
SMALL_F = 12                    # encoder width 36: heads 6 and 18 wide at 6 / 2 heads, neither a multiple of 4
SMALL = [f"{enc}_h{h}" for enc in ("AttnDIN", "DASALC", "AllRank") for h in (6, 2)]
SUBTOPICS = (6, 2, 4)


def case_config(name):
    """-> (F, listsf dict, list lengths) of a fixture case: ``<encoder>_h<heads>`` or ``default``."""
    if name == "default":
        return 100, dict(DEFAULT_LISTSF), (256, 2, 37)
    enc, h = name.split("_h")
    return SMALL_F, dict(SMALL_LISTSF, encoder_type=enc, n_heads=int(h)), (150, 2, 37)


def grad_query(name):
    """The query whose one-step parameter gradients the fixture holds (the file stays small): the 150-document list at 6
    heads, the 37-document one at 2 heads, none for the default.  A 2-document list is never one: a per-query BN over two
    rows outputs +-1 whatever they hold, so every gradient upstream of the last BN is 0 in exact arithmetic."""
    if name == "default":
        return None
    return 0 if name.endswith("_h6") else 2


def case_inputs(name, seed=2024):
    """[(q_repr [1,F], doc_reprs [n,F], subtopic relevance [m,n])] of a fixture case, rebuilt from (seed, name) so the
    fixture does not store them."""
    F, _, lens = case_config(name)
    rng = np.random.default_rng([seed, zlib.crc32(name.encode())])
    out = []
    for n, m in zip(lens, SUBTOPICS):
        q = rng.standard_normal((1, F)).astype(np.float32)
        d = rng.standard_normal((n, F)).astype(np.float32)
        R = (rng.random((m, n)) < 0.3).astype(np.float32)
        R[0, 0] = 1.0
        out.append((q, d, R))
    return out


def seeded_state(shapes, seed=4242):
    """{part: {key: float32 array}} for {part: {key: shape}} of a listsf checkpoint ('encoder', 'uni_sf'): Linear
    weights xavier-normal, LayerNorm gains and BN weights near 1, every other entry small."""
    out = {}
    for part, keys in shapes.items():
        out[part] = {}
        for key, shape in keys.items():
            rng = np.random.default_rng([seed, zlib.crc32(f"{part}.{key}".encode())])
            if len(shape) == 2:
                a = rng.standard_normal(shape) * np.sqrt(2.0 / (shape[0] + shape[1]))
            elif key.endswith("a_2") or key.endswith("bn.weight"):
                a = 1.0 + 0.1 * rng.standard_normal(shape)
            else:
                a = 0.1 * rng.standard_normal(shape)
            out[part][key] = a.astype(np.float32)
    return out


def state_shapes(encoder, uni_sf):
    return {"encoder": {k: tuple(v.shape) for k, v in encoder.state_dict().items()},
            "uni_sf": {k: tuple(v.shape) for k, v in uni_sf.state_dict().items()}}


def _encoder_key(key):
    """The reference encoder's state_dict key -> OracleDivList's."""
    key = key.replace("sublayer_cont.0.norm", "norm0").replace("sublayer_cont.1.norm", "norm1")
    key = key.replace("sublayer_cont.norm", "norm").replace(".fc.w1", ".w1").replace(".fc.w2", ".w2")
    return "final_norm" + key[4:] if key.startswith("norm.") else key


class OracleDivList(nn.Module):
    """Encoder of width 3F over [q, d, q*d] and uni_sf over [q, d, q*d, enc] for one query, in ATen ops (fp32).  The
    uni_sf BN (LTRBatchNorm on the reference's [n, 6F]) is the across-rows BN of a one-query [1, n, 6F] batch."""

    def __init__(self, num_features, n_heads, encoder_layers, encoder_type, ff_dims, AF='R', TL_AF='GE',
                 apply_tl_af=False, BN=True, bn_type='BN', bn_affine=False, dropout=0.1):
        super().__init__()
        W = 3 * num_features
        self.layers = nn.ModuleList([rp.RefEncoderLayer(W, n_heads, encoder_type, dropout)
                                     for _ in range(encoder_layers)])
        self.final_norm = rp.RefLayerNorm(W) if encoder_type == "AllRank" else None
        self.uni_sf = rp.stacked_ffnet([2 * W, *ff_dims, 1], AF, TL_AF, apply_tl_af, 0.1, BN, bn_type, bn_affine)

    def load_reference_state(self, encoder_sd, uni_sd):
        enc = {_encoder_key(k): torch.as_tensor(np.asarray(v)) for k, v in encoder_sd.items()}
        own = {k: v for k, v in self.state_dict().items() if not k.startswith("uni_sf.")}
        assert set(enc) == set(own), (sorted(set(enc) ^ set(own)))
        self.load_state_dict({**enc, **{"uni_sf." + k: torch.as_tensor(np.asarray(v)) for k, v in uni_sd.items()}})

    def forward(self, q_repr, doc_reprs):
        """q_repr [1,F] (or [F]), doc_reprs [n,F] -> [1,n] (div_list_ranker.py:61-85)."""
        q = q_repr.reshape(1, -1).expand(doc_reprs.size(0), -1)
        x = torch.cat((q, doc_reprs, q * doc_reprs), 1)
        z = x.unsqueeze(0)
        for layer in self.layers:
            z = layer(z)
        if self.final_norm is not None:
            z = self.final_norm(z)
        h = torch.cat((x, z[0]), 1).unsqueeze(0)
        return self.uni_sf(h).view(1, -1)


def reference_key_of(oracle_key):
    """OracleDivList parameter name -> (part, the reference's key)."""
    if oracle_key.startswith("uni_sf."):
        return "uni_sf", oracle_key[7:]
    k = oracle_key
    if k.startswith("final_norm."):
        return "encoder", "norm." + k[len("final_norm."):]
    for a, b in ((".norm0.", ".sublayer_cont.0.norm."), (".norm1.", ".sublayer_cont.1.norm."), (".w1.", ".fc.w1."),
                 (".w2.", ".fc.w2.")):
        if a in k:
            return "encoder", k.replace(a, b)
    if ".norm." in k:
        return "encoder", k.replace(".norm.", ".sublayer_cont.norm.")
    return "encoder", k
