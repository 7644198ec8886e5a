"""Attention pooling of the text encoder on the GPU: the latent cross-attention kernel against the projected form it
replaces, and the engine (`pooling="attention"`) against the oracle."""

import ctypes as C

import pytest
import torch

from oracle.text_attention_pooler import (OracleAttentionEncoderConfig, OracleAttentionTextEncoder,
                                         make_synthetic_attention_state_dict)
from tests.helpers import parity_metrics, rel_err

pytestmark = pytest.mark.gpu

VOCAB = 4096


def _bf(t):
    return t.to(torch.bfloat16).float()


@pytest.mark.parametrize("hd", [4, 16])
@pytest.mark.parametrize("lens", [[1, 17, 128, 514, 0, 3], "8200"])
def test_latent_kernel_matches_projected_attention(native_lib, cuda_device, hd, lens):
    """One query per sentence: K/V projection + SDPA (fp32 on bf16-rounded inputs) against the kernel on the absorbed
    form (qt_h = W_k,h^T q_h, then W_v,h u_h + b_v,h).  8200 sentences put cu_seqlens beyond any small staging."""
    from sonar_b200 import ops

    g = torch.Generator().manual_seed(hd)
    if lens == "8200":
        lens = torch.randint(0, 40, (8200,), generator=g).tolist()
        lens[5] = 0
    d, e = 1024, 64 * hd
    b = len(lens)
    mem = _bf(torch.randn(sum(lens), d, generator=g))
    wk, wv = _bf(torch.randn(e, d, generator=g) * d ** -0.5), _bf(torch.randn(e, d, generator=g) * d ** -0.5)
    bk, bv = torch.randn(e, generator=g) * 0.1, torch.randn(e, generator=g) * 0.1
    q = torch.randn(b, e, generator=g) * 2.0
    qt = torch.einsum("bhj,hjd->bhd", q.view(b, hd, 64), wk.view(hd, 64, d)).contiguous()
    cu = ops.cu_seqlens_of(lens)
    u = ops.pool_latent_attention(qt.to(torch.bfloat16).to(cuda_device), mem.to(torch.bfloat16).to(cuda_device),
                                  cu.to(cuda_device)).float().cpu()
    got = torch.einsum("hjd,bhd->bhj", wv.view(hd, 64, d), u).reshape(b, e) + bv
    qb = _bf(qt)  # the kernel's rounded queries; the projected form below reads the same scores up to q . b_k
    for i, n in enumerate(lens):
        s0, s1 = int(cu[i]), int(cu[i + 1])
        if n == 0:
            assert torch.equal(u[i], torch.zeros_like(u[i])), i
            continue
        if i > 64 and n != max(lens):  # the long 8200 case: check a sample plus the longest sentence
            continue
        k = (mem[s0:s1] @ wk.T + bk).view(n, hd, 64)
        v = (mem[s0:s1] @ wv.T + bv).view(n, hd, 64)
        att = torch.softmax(torch.einsum("hj,thj->ht", q[i].view(hd, 64), k) / 8.0, dim=-1)
        ref = torch.einsum("ht,thj->hj", att, v).reshape(e)
        assert rel_err(got[i], ref) <= 2e-2, (i, n, rel_err(got[i], ref))
        lat = torch.softmax(qb[i] @ mem[s0:s1].T / 8.0, dim=-1) @ mem[s0:s1]
        assert rel_err(u[i], lat) <= 1e-2, (i, n, rel_err(u[i], lat))


def _build(num_layers, pooler_layers, device, embedding_dim=None, ln_fold=0, seed=1, pooler_std=0.02):
    from sonar_b200 import B200TextEncoderModel, VocabularyInfo, sonar_text_encoder_config

    e = embedding_dim or 1024
    ocfg = OracleAttentionEncoderConfig(vocab_size=VOCAB, num_layers=num_layers, embedding_dim=embedding_dim,
                                        pooler_layers=pooler_layers, pooler_heads=e // 64)
    sd = make_synthetic_attention_state_dict(ocfg, seed=seed, pooler_std=pooler_std)
    cfg = sonar_text_encoder_config(
        "basic", num_encoder_layers=num_layers, num_decoder_layers=pooler_layers, num_decoder_attn_heads=e // 64,
        pooling="attention", embedding_dim=embedding_dim,
        vocab_info=VocabularyInfo(size=VOCAB, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1))
    return OracleAttentionTextEncoder(ocfg, sd), B200TextEncoderModel(cfg, sd, device, ln_fold=ln_fold), sd


def _batch(lens, s, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros((len(lens), s), dtype=torch.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(4, VOCAB, (n,), generator=g)
    return ids


def _check(m, what):
    print(what, m)
    assert m["one_minus_cos_max"] <= 1e-3, (what, m)
    assert m["centred_cos_min"] >= 0.999, (what, m)
    assert m["rel_l2_max"] <= 1e-2, (what, m)


def _run(model, ids, lens, device):
    from sonar_b200 import PaddingMask, SequenceBatch

    s = ids.shape[1]
    return model(SequenceBatch(ids.to(device), PaddingMask(torch.tensor(lens), s, lens)))


LENS = [514, 1, 2, 17, 33, 300, 48, 5, 128, 31, 16, 8]


@pytest.mark.parametrize("embedding_dim", [None, 256])
def test_two_layer_pooler_vs_oracle(native_lib, cuda_device, embedding_dim):
    oracle, _, sd = _build(2, 2, cuda_device, embedding_dim)
    ids = _batch(LENS, 514, seed=3)
    ref, _ = oracle(ids, torch.tensor(LENS))
    for ln_fold in (0, 1, 2):
        _, model, _ = _build(2, 2, cuda_device, embedding_dim, ln_fold=ln_fold)
        out = _run(model, ids, LENS, cuda_device).sentence_embeddings
        assert out.shape == (len(LENS), embedding_dim or 1024)
        _check(parity_metrics(out, ref), f"E={embedding_dim} ln_fold={ln_fold}")


def test_full_basic_shape_vs_oracle(native_lib, cuda_device):
    """BASELINE.json config 1 batch (32 sentences, lengths U{8..64}) through 24 encoder and 24 pooler layers.  With the
    default std-0.02 pooler weights, 24 POST-LN layers wash the sentence out of the oracle's embeddings (mean pairwise
    cosine 0.97), so the mean-centred metrics would only measure bf16 noise; std-0.05 pooler weights keep them apart."""
    oracle, model, _ = _build(24, 24, cuda_device, pooler_std=0.05)
    g = torch.Generator().manual_seed(0)
    lens = torch.randint(8, 65, (32,), generator=g).tolist()
    ids = _batch(lens, 64, seed=5)
    ref, _ = oracle(ids, torch.tensor(lens))
    _check(parity_metrics(_run(model, ids, lens, cuda_device).sentence_embeddings, ref), "24+24 layers")


@pytest.fixture(scope="module")
def small(native_lib, cuda_device):
    return _build(2, 2, cuda_device, 256)


def test_batch_composition_invariance_bitwise(small, cuda_device):
    from sonar_b200 import SequenceBatch

    _, model, _ = small
    lens = [40, 7, 64, 23, 64, 1]
    ids = _batch(lens, 64, seed=6)
    full = _run(model, ids, lens, cuda_device).sentence_embeddings
    for i, n in enumerate(lens):
        one = model(SequenceBatch(ids[i : i + 1, :n].contiguous().to(cuda_device), None)).sentence_embeddings
        assert torch.equal(one[0], full[i]), i


def test_encoded_seqs_do_not_depend_on_the_pooling(small, cuda_device):
    from sonar_b200 import B200TextEncoderModel, VocabularyInfo, sonar_text_encoder_config

    _, attn, sd = small
    cfg = sonar_text_encoder_config("basic", num_encoder_layers=2,
                                    vocab_info=VocabularyInfo(size=VOCAB, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1))
    mean = B200TextEncoderModel(cfg, sd, cuda_device)
    lens = [17, 1, 64, 30]
    ids = _batch(lens, 64, seed=7)
    attn.return_encoded_seqs = mean.return_encoded_seqs = True
    try:
        a, m = _run(attn, ids, lens, cuda_device), _run(mean, ids, lens, cuda_device)
    finally:
        attn.return_encoded_seqs = False
    assert torch.equal(a.encoded_seqs, m.encoded_seqs)
    assert a.sentence_embeddings.shape == (4, 256) and m.sentence_embeddings.shape == (4, 1024)


def test_predict_preserves_order_and_width(small, cuda_device):
    from sonar_b200.inference_pipelines import TextToEmbeddingModelPipeline
    from sonar_b200.tokenizer import SyntheticTokenizer

    oracle, model, _ = small
    pipe = TextToEmbeddingModelPipeline(model, SyntheticTokenizer(vocab_size=VOCAB), device=cuda_device)
    sents = ["the quick brown fox", "a", "jumps over the lazy dog again and again", "hello world", "b c"]
    emb = pipe.predict(sents, source_lang="eng_Latn", batch_size=2)
    assert emb.shape == (len(sents), 256)
    enc = pipe.tokenizer.create_encoder(lang="eng_Latn")
    for i, s in enumerate(sents):
        ref, _ = oracle(enc(s)[None], None)
        m = parity_metrics(emb[i : i + 1], ref)
        assert m["one_minus_cos_max"] <= 1e-3 and m["rel_l2_max"] <= 1e-2, (i, m)


def test_forward_host_and_small_workspace(small, cuda_device):
    from sonar_b200 import _lib

    _, model, _ = small
    lib, dev = model._lib, cuda_device
    lens = [9, 3]
    ids = _batch(lens, 16, seed=8)
    want = _run(model, ids, lens, dev).sentence_embeddings.cpu()
    lens_c = (C.c_int32 * 2)(*lens)
    out_host = torch.empty((2, 256), dtype=torch.float32)
    ids_host = ids.contiguous()
    staging_ids = torch.empty(2 * 16, dtype=torch.int64, device=dev)
    staging_out = torch.empty(2 * 256, dtype=torch.float32, device=dev)
    ws = model._ensure_workspace(2, 12)
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        rc = lib.sb_encoder_forward_host(model._handle, ids_host.data_ptr(), lens_c, 2, 16, out_host.data_ptr(),
                                         staging_ids.data_ptr(), staging_out.data_ptr(), ws.data_ptr(), ws.numel(), stream)
    _lib.check(rc, "sb_encoder_forward_host")
    assert torch.equal(out_host, want)
    tiny = torch.zeros(1, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = lib.sb_encoder_forward(model._handle, ids.to(dev).data_ptr(), 16, lens_c, 2, 16, staging_out.data_ptr(), None,
                                    tiny.data_ptr(), 1, stream)
    assert rc == _lib.SB_ERR_INVALID
    assert _lib.last_error().startswith("sb_encoder_forward: workspace too small")
    torch.cuda.synchronize(dev)
