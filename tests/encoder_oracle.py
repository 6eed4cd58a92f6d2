"""fp32 numpy restatement of ctranslate2::Encoder on a TransformerEncoderSpec model, built on the encoder layers of
oracle.ct2_oracle.Seq2SeqOracle (its Dense, LayerNorm, sublayer and attention helpers).

Reference: models::EncoderReplica::forward_impl (src/models/language_model.cc:349-400: token-type placeholder of zeros,
pooler_dense + pooler_activation on the first position), TransformerEncoder::operator() (src/layers/transformer.cc:427-471:
merged embeddings, embedding scale, position encoder, layernorm_embedding, the layers, output norm), ParallelEmbeddings
(src/layers/common.cc:116-148: ADD merge)."""
from __future__ import annotations

import json
import math
import os
import struct
from typing import Dict, Optional

import numpy as np

from oracle import ct2_oracle as O

f32 = np.float32


def load_fixture(path: str) -> Dict:
    """tests/golden/encoder_ref.npz (tools/make_golden.py --encoder-only) as {model: [case]}, each case a dict with
    compute_type, ids / token_type_ids (lists of the valid positions, types None when not given), last_hidden_state (one
    flattened [len * d] array per row) and pooler_output ([B, d] or None)."""
    z = np.load(path)
    fixture: Dict = {}
    k = 0
    while f"c{k}_model" in z:
        c = f"c{k}_"
        lens = z[c + "lens"]
        rows = lambda a: [a[b, :n].tolist() for b, n in enumerate(lens)]     # noqa: E731
        hidden = np.split(z[c + "hidden"], np.cumsum(lens)[:-1])
        fixture.setdefault(str(z[c + "model"]), []).append({
            "compute_type": str(z[c + "compute"]), "ids": rows(z[c + "ids"]),
            "token_type_ids": rows(z[c + "types"]) if c + "types" in z else None,
            "last_hidden_state": [h.reshape(-1) for h in hidden],
            "pooler_output": z[c + "pooled"] if c + "pooled" in z else None})
        k += 1
    return fixture


class EncoderOracle(O.Seq2SeqOracle):
    def __init__(self, variables: Dict[str, np.ndarray], compute_type: str = "float32", flavor: str = "cpu",
                 binary_version: int = 6, eps: float = 1e-5):
        # the attributes the Seq2SeqOracle encoder helpers read; there is no decoder to describe
        self.v = variables
        self.flavor = flavor
        self.round_before_cast = binary_version >= 5
        self.compute_type = compute_type
        self._float_w = {}
        self.num_heads = int(variables.get("encoder/num_heads", np.int16(8)))
        self.enc_emb = "encoder/embeddings_0" if "encoder/embeddings_0/weight" in variables else "encoder/embeddings"
        self.d = variables[self.enc_emb + "/weight"].shape[1]
        self.enc_layers = 0
        while f"encoder/layer_{self.enc_layers}/ffn/linear_0/weight" in variables:
            self.enc_layers += 1
        self.pos = variables["encoder/position_encodings/encodings"].astype(f32)
        self.pre_norm = {"encoder": bool(variables.get("encoder/pre_norm", True))}
        self.act = {"encoder": int(variables.get("encoder/activation", O.ACT_RELU))}
        sc = variables.get("encoder/scale_embeddings")                # build_embeddings_scale, transformer.cc:380-402
        if sc is None or (sc.dtype == np.int8 and bool(sc)):
            self.scale = f32(math.sqrt(self.d))
        elif sc.dtype != np.int8 and float(sc) != 1.0:
            self.scale = f32(sc)
        else:
            self.scale = None
        self.eps = eps

    @classmethod
    def from_dir(cls, model_dir: str, compute_type: str = "float32", flavor: str = "cpu") -> "EncoderOracle":
        _, _, variables, _ = O.read_model_bin(model_dir + "/model.bin")
        with open(model_dir + "/model.bin", "rb") as f:
            binary_version = struct.unpack("<I", f.read(4))[0]
        eps = 1e-5
        cfg = os.path.join(model_dir, "config.json")
        if os.path.exists(cfg):
            with open(cfg) as f:
                e = json.load(f).get("layer_norm_epsilon")
            eps = eps if e is None else float(e)
        return cls(variables, compute_type=compute_type, flavor=flavor, binary_version=binary_version, eps=eps)

    def _table(self, prefix: str, ids: np.ndarray) -> np.ndarray:
        """Embeddings::operator() (common.cc:64-81): gather, int8 rows divided by their scale."""
        x = O.gather_rows(self.v[prefix + "/weight"], ids).astype(f32)
        if prefix + "/weight_scale" in self.v:
            sc = self.v[prefix + "/weight_scale"].astype(f32)
            x = (x / (O.gather_rows(sc, ids)[..., None] if sc.ndim == 1 else sc)).astype(f32)
        return x

    def forward(self, ids: np.ndarray, lengths: np.ndarray, token_type_ids: Optional[np.ndarray] = None):
        """ids [B, T] (padding ignored through lengths) -> (last_hidden_state [B, T, d], pooler_output [B, d] or None)."""
        B, T = ids.shape
        x = self._table(self.enc_emb, ids)
        if "encoder/embeddings_1/weight" in self.v:                   # token types, zeros when not given
            types = np.zeros_like(ids) if token_type_ids is None else token_type_ids
            x = (self._table("encoder/embeddings_1", types) + x).astype(f32)
        if self.scale is not None:
            x = (x * self.scale).astype(f32)
        x = (x + self.pos[:T][None]).astype(f32)
        if "encoder/layernorm_embedding/gamma" in self.v:
            x = self._ln("encoder/layernorm_embedding", x)
        lens_rows = np.repeat(np.asarray(lengths), self.num_heads * T)
        for l in range(self.enc_layers):
            p = f"encoder/layer_{l}/"

            def attn(h, res):
                q, k, v_ = np.split(self._dense(p + "self_attention/linear_0", h), 3, axis=-1)
                return self._dense(p + "self_attention/linear_1", self._attend(q, k, v_, lens_rows), residual=res)

            def ffn(h, res):
                return self._dense(p + "ffn/linear_1", self._dense(p + "ffn/linear_0", h, act=self.act["encoder"]), residual=res)

            x = self._sublayer("encoder", p + "self_attention", x, attn)
            x = self._sublayer("encoder", p + "ffn", x, ffn)
        if "encoder/layer_norm/gamma" in self.v:
            x = self._ln("encoder/layer_norm", x)
        pooled = None
        if "pooler_dense/weight" in self.v:
            pooled = self._dense("pooler_dense", x[:, 0], act=int(self.v.get("pooler_activation", O.ACT_TANH)))
        return x, pooled
