"""Attention pooling of the text encoder without a GPU: the oracle's pooler against an independent composition of torch
modules and against the HuggingFace-pinned golden, the reference's low-dimension encoder test restated on the oracle,
the config envelope of the CUDA wrapper, and the ctypes mirror of the C structs."""

import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle.text_attention_pooler import (OracleAttentionEncoderConfig, OracleAttentionTextEncoder,
                                         make_synthetic_attention_state_dict)
from oracle.text_encoder import OracleEncoderConfig, make_synthetic_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torch_pooler(sd, cfg, enc, key_ok):
    """The attention pooler from torch.nn.MultiheadAttention / LayerNorm / Linear modules (fp64)."""
    e, d, h = cfg.out_dim, cfg.model_dim, cfg.pooler_heads
    fp = cfg.pooler_ffn_inner_dim or cfg.ffn_inner_dim
    kw = dict(dtype=torch.float64)

    def attn(pfx, kdim):
        m = torch.nn.MultiheadAttention(e, h, kdim=kdim, vdim=kdim, batch_first=True, **kw)
        q, k, v = (sd[pfx + f"{n}_proj.weight"].double() for n in ("q", "k", "v"))
        if m._qkv_same_embed_dim:
            m.in_proj_weight.data.copy_(torch.cat([q, k, v], 0))
        else:
            m.q_proj_weight.data.copy_(q)
            m.k_proj_weight.data.copy_(k)
            m.v_proj_weight.data.copy_(v)
        m.in_proj_bias.data.copy_(torch.cat([sd[pfx + f"{n}_proj.bias"].double() for n in ("q", "k", "v")]))
        m.out_proj.weight.data.copy_(sd[pfx + "output_proj.weight"].double())
        m.out_proj.bias.data.copy_(sd[pfx + "output_proj.bias"].double())
        return m

    def ln(name):
        m = torch.nn.LayerNorm(e, eps=cfg.ln_eps, **kw)
        m.weight.data.copy_(sd[name + ".weight"].double())
        m.bias.data.copy_(sd[name + ".bias"].double())
        return m

    def lin(name, i, o):
        m = torch.nn.Linear(i, o, **kw)
        m.weight.data.copy_(sd[name + ".weight"].double())
        m.bias.data.copy_(sd[name + ".bias"].double())
        return m

    b = enc.shape[0]
    pos0 = torch.cat([torch.zeros(e // 2), torch.ones(e - e // 2)]).double()
    x = (sd["pooler.decoder_frontend.embed.weight"][0].double() * e ** 0.5 + pos0).expand(b, 1, e)
    enc = enc.double()
    with torch.no_grad():
        for i in range(cfg.pooler_layers):
            p = f"pooler.decoder.layers.{i}."
            x = ln(p + "self_attn_layer_norm")(x + attn(p + "self_attn.", e)(x, x, x, need_weights=False)[0])
            ca = attn(p + "encoder_decoder_attn.", d)(x, enc, enc, key_padding_mask=~key_ok, need_weights=False)[0]
            x = ln(p + "encoder_decoder_attn_layer_norm")(x + ca)
            f = lin(p + "ffn.output_proj", fp, e)(torch.relu(lin(p + "ffn.inner_proj", e, fp)(x)))
            x = ln(p + "ffn_layer_norm")(x + f)
        return lin("pooler.projection_out", e, e)(x).squeeze(1)


@pytest.mark.parametrize("model_dim,embedding_dim", [(64, None), (64, 128), (128, 64)])
def test_oracle_pooler_matches_torch_modules(model_dim, embedding_dim):
    cfg = OracleAttentionEncoderConfig(model_dim=model_dim, vocab_size=50, num_layers=1, num_heads=4, ffn_inner_dim=96,
                                       embedding_dim=embedding_dim, pooler_layers=2, pooler_heads=4,
                                       pooler_ffn_inner_dim=80)
    sd = make_synthetic_attention_state_dict(cfg, seed=5, weight_std=0.1)
    oracle = OracleAttentionTextEncoder(cfg, sd, dtype=torch.float64)
    lens = torch.tensor([7, 1, 4, 3])
    g = torch.Generator().manual_seed(0)
    enc = torch.randn(len(lens), 7, model_dim, generator=g, dtype=torch.float64)
    key_ok = torch.arange(7)[None, :] < lens[:, None]
    got = oracle.pooler(enc, key_ok)
    ref = _torch_pooler(sd, cfg, enc, key_ok)
    assert got.shape == (len(lens), cfg.out_dim)
    assert float((got - ref).abs().max()) <= 1e-10
    # and through the whole forward: the pooler sees the final-LayerNormed states of the real tokens only
    ids = torch.randint(4, 50, (len(lens), 7), generator=g)
    emb, x = oracle(ids, lens)
    assert float((emb - _torch_pooler(sd, cfg, x, key_ok)).abs().max()) <= 1e-10


def test_oracle_pooler_layers_match_the_hf_golden():
    """E = D: the text oracle's pooler layers against the HuggingFace BartDecoderLayer golden of the speech pooler."""
    g = torch.load(os.path.join(ROOT, "tests", "golden", "pooler_layers_small.pt"), weights_only=True)
    c = g["config"]
    cfg = OracleAttentionEncoderConfig(model_dim=c["model_dim"], num_layers=0, pooler_layers=c["pooler_layers"],
                                       pooler_heads=c["pooler_heads"], pooler_ffn_inner_dim=c["pooler_ffn_inner_dim"])
    sd = {k.replace("encoder_pooler.", "pooler."): v for k, v in g["state_dict"].items()}
    oracle = OracleAttentionTextEncoder(cfg, sd)
    key_ok = torch.arange(g["enc"].shape[1])[None, :] < g["lens"][:, None]
    torch.testing.assert_close(oracle.pooler_layers(g["x0"], g["enc"], key_ok), g["out"], rtol=1e-5, atol=1e-5)


def test_low_dim_encoder_on_the_oracle():
    """The reference's tests/unit_tests/test_low_dimension_text_models.py::test_low_dim_encoder: a `basic` encoder with
    model_dim 32, embedding_dim 256, 5 encoder and 2 pooler layers and attention pooling maps 3 sentences to (3, 256)."""
    cfg = OracleAttentionEncoderConfig(model_dim=32, num_layers=5, embedding_dim=256, pooler_layers=2)
    oracle = OracleAttentionTextEncoder(cfg, make_synthetic_attention_state_dict(cfg, seed=1))
    emb, _ = oracle(torch.tensor([[0, 1, 2, 3, 4]] * 3), None)
    assert emb.shape == (3, 256) and bool(torch.isfinite(emb).all())


def test_pooler_weights_leave_the_encoder_weights_alone():
    base = OracleEncoderConfig(model_dim=64, vocab_size=50, num_layers=2, num_heads=4, ffn_inner_dim=128)
    plain = make_synthetic_state_dict(base, seed=3)
    attn = make_synthetic_attention_state_dict(OracleAttentionEncoderConfig(**base.__dict__, pooler_layers=1,
                                                                            pooler_heads=4), seed=3)
    assert all(torch.equal(plain[k], attn[k]) for k in plain)
    assert set(attn) - set(plain) and all(k.startswith("pooler.") for k in set(attn) - set(plain))


def test_check_supported_envelope():
    from sonar_b200.text_encoder import _check_supported, sonar_text_encoder_config

    ok = [dict(), dict(pooling="attention"), dict(pooling="attention", embedding_dim=256, num_decoder_attn_heads=4),
          dict(pooling="attention", embedding_dim=1024), dict(pooling="attention", decoder_ffn_inner_dim=4096),
          dict(pooling="max", embedding_dim=1024)]
    bad = [dict(pooling="mean", embedding_dim=256), dict(pooling="attention", embedding_dim=256),  # 16 heads of 16
           dict(pooling="attention", embedding_dim=2048, num_decoder_attn_heads=32),
           dict(pooling="attention", embedding_dim=320, num_decoder_attn_heads=5),
           dict(pooling="attention", decoder_ffn_inner_dim=1000), dict(pooling="attention", num_decoder_layers=0),
           dict(pooling="attention", normalize_before=True), dict(pooling="median")]
    for o in ok:
        _check_supported(sonar_text_encoder_config("basic", **o))
    for o in bad:
        with pytest.raises(NotImplementedError):
            _check_supported(sonar_text_encoder_config("basic", **o))


def _header_fields(header, name):
    body = re.search(r"typedef struct " + name + r" \{(.*?)\} " + name + ";", header, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"(\w+)\s*(?:/\*.*?\*/\s*)?;", body)


@pytest.mark.parametrize("name", ["SbEncoderConfig", "SbEncoderWeights", "SbPoolerLayerWeights"])
def test_ctypes_structs_match_the_header(name, tmp_path):
    from sonar_b200 import _lib

    header = open(os.path.join(ROOT, "include", "sonar_b200.h")).read()
    struct = getattr(_lib, name)
    assert [f for f, _ in struct._fields_] == _header_fields(header, name)
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler to measure the C layout")
    src = tmp_path / "layout.c"
    fields = [f for f, _ in struct._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sonar_b200.h"\nint main(void) {\n'
                   f'  printf("%zu\\n", sizeof({name}));\n' +
                   "".join(f'  printf("%zu\\n", offsetof({name}, {f}));\n' for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(struct)] + [getattr(struct, f).offset for f in fields]
