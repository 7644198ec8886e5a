"""GPU tests of the LASER2 text encoder: the LSTM recurrent kernel against a torch recurrence, the engine against the
float64 oracle at the `laser2` shape, bitwise batch invariance, order, the reference's masking, and input errors."""

import ctypes as C

import pytest
import torch

from oracle.laser_lstm import OracleLaser2, OracleLaser2Config, make_synthetic_laser2_state_dict

pytestmark = pytest.mark.gpu

H = 512
# LSTM weights U(-0.1, 0.1) (torch's default bound is 1/sqrt(512) = 0.044): with the default, 5 layers leave every
# sentence's max-pooled embedding within 0.985-0.997 cosine of every other's; with 0.1 the off-diagonal range is about
# 0.6-0.9 (printed by test_engine_matches_the_oracle), so the tolerances below separate sentences.
WEIGHT_BOUND = 0.1


def _rows(dirs):
    from sonar_b200.ops import lstm_gate_rows

    return lstm_gate_rows(H, dirs)


def _torch_recurrence(g_nat, w_hh_nat, lens, dirs, round_h):
    """fp32 LSTM recurrence over packed tokens in torch.nn.LSTM's gate order: g_nat [T, dirs*4H] input pre-activations,
    w_hh_nat [dirs*4H, H] -> y [T, dirs*H]; with round_h the matmul reads bf16(h), as the kernel does."""
    dev = g_nat.device
    lens_t = torch.tensor(lens, device=dev)
    cu = torch.zeros(len(lens) + 1, dtype=torch.int64, device=dev)
    cu[1:] = torch.cumsum(lens_t, 0)
    y = torch.zeros(g_nat.shape[0], dirs * H, device=dev)
    rows = torch.arange(len(lens), device=dev)
    for d in range(dirs):
        w = w_hh_nat[d * 4 * H:(d + 1) * 4 * H].float()
        h = torch.zeros(len(lens), H, device=dev)
        c = torch.zeros(len(lens), H, device=dev)
        for s in range(max(lens)):
            idx = rows[lens_t > s]
            tok = cu[idx] + (lens_t[idx] - 1 - s if d else s)
            hin = h[idx].bfloat16().float() if round_h else h[idx]
            z = g_nat[tok, d * 4 * H:(d + 1) * 4 * H].float() + hin @ w.T
            zi, zf, zg, zo = z.split(H, dim=1)
            c[idx] = torch.sigmoid(zf) * c[idx] + torch.sigmoid(zi) * torch.tanh(zg)
            h[idx] = torch.sigmoid(zo) * torch.tanh(c[idx])
            y[tok, d * H:(d + 1) * H] = h[idx]
    return y, cu


@pytest.mark.parametrize("dirs", [1, 2])
def test_lstm_recurrent_kernel_against_torch(native_lib, cuda_device, dirs):
    from sonar_b200 import ops

    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(dirs)
    # 70 sequences: a full tile of mixed lengths (the order below is not sorted) and a tile of 6 rows
    lens = torch.randint(1, 90, (70,), generator=g).tolist()
    lens[3], lens[40] = 1, 130
    T = sum(lens)
    g_nat = (torch.randn(T, dirs * 4 * H, generator=g) * 0.7).bfloat16().to(cuda_device)
    w_nat = ((torch.rand(dirs * 4 * H, H, generator=g) * 2 - 1) * WEIGHT_BOUND).bfloat16().to(cuda_device)
    rows = _rows(dirs).to(cuda_device)
    tiles = torch.full((128,), -1, dtype=torch.int32)
    tiles[:70] = torch.randperm(70, generator=g).to(torch.int32)
    tiles = tiles.to(cuda_device)
    y_ref, cu = _torch_recurrence(g_nat, w_nat, lens, dirs, round_h=True)
    y_f32, _ = _torch_recurrence(g_nat, w_nat, lens, dirs, round_h=False)
    cu32 = cu.to(torch.int32)
    y = ops.lstm_recurrent(g_nat[:, rows].contiguous(), w_nat[rows].contiguous(), cu32, tiles, dirs)
    torch.cuda.synchronize()
    err = (y.float() - y_ref).abs().max().item()
    err32 = (y.float() - y_f32).abs().max().item()
    print(f"dirs={dirs}: max |y - ref(bf16 h)| = {err:.3e}, max |y - ref(fp32 h)| = {err32:.3e}")
    assert err <= 1.5e-2 and err32 <= 5e-2

    # the pooling variant: pad tokens skipped, the tail's padding value where flagged
    pad = (torch.rand(T, generator=g) < 0.1).to(torch.uint8).to(cuda_device)
    tail = (torch.rand(70, generator=g) < 0.5).to(torch.uint8).to(cuda_device)
    pooled = ops.lstm_recurrent(g_nat[:, rows].contiguous(), w_nat[rows].contiguous(), cu32, tiles, dirs, pool=True,
                                pad_mask=pad, tail_keep=tail, padding_value=0.25)
    want = torch.full((70, dirs * H), float("-inf"), device=cuda_device)
    for b in range(70):
        seg = y_ref[cu[b]:cu[b + 1]][pad[cu[b]:cu[b + 1]] == 0]
        if seg.shape[0]:
            want[b] = seg.max(0).values
        if tail[b]:
            want[b] = torch.clamp(want[b], min=0.25)
    fin = torch.isfinite(want)
    assert torch.equal(fin, torch.isfinite(pooled))
    assert (pooled[fin] - want[fin]).abs().max().item() <= 1.5e-2


def _model(cfg, seed=1, device="cuda:0"):
    from sonar_b200 import B200LaserLstmEncoder, Laser2Config

    sd = make_synthetic_laser2_state_dict(cfg, seed=seed, weight_bound=WEIGHT_BOUND)
    lcfg = Laser2Config(vocabulary_size=cfg.vocabulary_size, pad_idx=cfg.pad_idx, model_dim=cfg.model_dim,
                        hidden_size=cfg.hidden_size, num_layers=cfg.num_layers, bidirectional=cfg.bidirectional,
                        padding_value=cfg.padding_value)
    return B200LaserLstmEncoder(lcfg, sd, device), sd


@pytest.fixture(scope="module")
def laser2(native_lib, cuda_device):
    cfg = OracleLaser2Config()  # the `laser2` shape: vocab 50004, 320 -> 5 x bidirectional 512
    model, sd = _model(cfg, device=cuda_device)
    return cfg, model, OracleLaser2(cfg, sd, dtype=torch.float64, device=cuda_device)


def _batch(lens, vocab, pad, seed, S=None):
    g = torch.Generator().manual_seed(seed)
    S = S or max(lens)
    ids = torch.full((len(lens), S), pad, dtype=torch.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(3, vocab, (n,), generator=g)
    return ids, torch.tensor(lens)


def _compare(got, ref, label):
    got, ref = got.double().cpu(), ref.double().cpu()
    cos = torch.nn.functional.cosine_similarity(got, ref, dim=1)
    mu = ref.mean(0, keepdim=True)
    ccos = torch.nn.functional.cosine_similarity(got - mu, ref - mu, dim=1)
    rel = (got - ref).norm(dim=1) / ref.norm(dim=1)
    n = torch.nn.functional.normalize(ref, dim=1)
    off = (n @ n.T)[~torch.eye(ref.shape[0], dtype=torch.bool)]
    print(f"{label}: 1-cos max {float((1 - cos).max()):.2e}, centred cos min {float(ccos.min()):.5f}, rel-L2 max "
          f"{float(rel.max()):.2e}; oracle off-diagonal cosines {float(off.min()):.3f}..{float(off.max()):.3f}")
    assert float((1 - cos).max()) <= 1e-3 and float(ccos.min()) >= 0.999 and float(rel.max()) <= 1e-2


@pytest.mark.parametrize("batch", [96, 1100])
def test_engine_matches_the_oracle(laser2, batch):
    """Lengths U{1..128} plus one 1024-token sentence; 96 sentences fill fewer clusters than the GPU holds at once, 1100
    several waves of them."""
    cfg, model, oracle = laser2
    g = torch.Generator().manual_seed(batch)
    lens = torch.randint(1, 129, (batch,), generator=g).tolist()
    lens[batch // 2] = 1024
    ids, lens_t = _batch(lens, cfg.vocabulary_size, cfg.pad_idx, seed=batch)
    got = model(ids.cuda(), lens_t)
    torch.cuda.synchronize()
    model.check_inputs()
    ref = oracle(ids, lens_t)
    _compare(got, ref, f"laser2 B={batch}")


def test_batch_composition_invariance_and_order(laser2):
    cfg, model, _ = laser2
    ids, lens = _batch([57], cfg.vocabulary_size, cfg.pad_idx, seed=7)
    alone = model(ids.cuda(), lens)
    for n, seed in ((5, 1), (64, 2), (300, 3)):
        g = torch.Generator().manual_seed(seed)
        other = torch.randint(1, 129, (n,), generator=g).tolist()
        o_ids, o_lens = _batch(other, cfg.vocabulary_size, cfg.pad_idx, seed=seed, S=128)
        at = n // 2
        o_ids[at] = cfg.pad_idx
        o_ids[at, :57] = ids[0]
        o_lens[at] = 57
        out = model(o_ids.cuda(), o_lens)
        assert torch.equal(out[at], alone[0]), f"batch of {n}"
        perm = torch.randperm(n, generator=g)
        out_p = model(o_ids[perm].cuda(), o_lens[perm])
        assert torch.equal(out_p, out[perm.cuda()]), "outputs follow the input order"


def test_masking_quirks_match_the_oracle(laser2):
    """A pad id inside a sentence is masked; padding with an id other than pad_idx contributes 0.0; a sentence whose
    positions are all pad ids pools to -inf, as in the reference."""
    cfg, model, oracle = laser2
    lens = [12, 5, 9, 3, 12]
    ids, lens_t = _batch(lens, cfg.vocabulary_size, cfg.pad_idx, seed=11)
    ids[0, 4] = cfg.pad_idx      # inside the sentence
    ids[1, 5:] = 0               # padded with id 0: 0.0 takes part in the max
    ids[3, :] = cfg.pad_idx      # every position is a pad id
    got = model(ids.cuda(), lens_t).cpu().double()
    ref = oracle(ids, lens_t).cpu()
    assert torch.equal(torch.isinf(got), torch.isinf(ref)) and bool(torch.isinf(got[3]).all())
    fin = [0, 1, 2, 4]
    _compare(got[fin], ref[fin], "masking")
    assert bool((got[1] >= 0).all())


def test_unidirectional_single_layer_matches_the_oracle(native_lib, cuda_device):
    cfg = OracleLaser2Config(vocabulary_size=1000, model_dim=128, num_layers=1, bidirectional=False)
    model, sd = _model(cfg, seed=2, device=cuda_device)
    ids, lens = _batch(torch.randint(1, 60, (80,), generator=torch.Generator().manual_seed(0)).tolist(),
                       cfg.vocabulary_size, cfg.pad_idx, seed=12)
    got = model(ids.cuda(), lens)
    assert got.shape == (80, 512)
    _compare(got, OracleLaser2(cfg, sd, device=cuda_device)(ids, lens), "1 layer, forward only")


def test_input_errors(laser2):
    cfg, model, _ = laser2
    ids, lens = _batch([4, 3], cfg.vocabulary_size, cfg.pad_idx, seed=13)
    with pytest.raises(RuntimeError, match="CUDA"):
        model(ids, lens)
    with pytest.raises(ValueError, match="seq_lens"):
        model(ids.cuda(), torch.tensor([4, 0]))
    bad = ids.clone()
    bad[1, 0] = cfg.vocabulary_size
    model(bad.cuda(), lens)
    with pytest.raises(ValueError, match="vocab"):
        model.check_inputs()
    model(ids.cuda(), lens)
    model.check_inputs()  # the flag was cleared by the failed check
    tiny = torch.empty(1, dtype=torch.uint8, device="cuda")
    out = torch.empty(2, 1024, device="cuda")
    d_ids = ids.cuda()
    lens_c = (C.c_int32 * 2)(4, 3)
    from sonar_b200 import _lib

    rc = model._lib.sb_laser2_forward(model._handle, d_ids.data_ptr(), d_ids.stride(0), lens_c, 2, 4, out.data_ptr(),
                                      tiny.data_ptr(), 1, torch.cuda.current_stream().cuda_stream)
    with pytest.raises(ValueError, match="workspace too small"):
        _lib.check(rc, "sb_laser2_forward")


def test_envelope_errors(native_lib, cuda_device):
    from sonar_b200 import B200LaserLstmEncoder, laser2_config

    with pytest.raises(NotImplementedError, match="hidden_size"):
        B200LaserLstmEncoder(laser2_config(hidden_size=256), {}, cuda_device)
    with pytest.raises(RuntimeError, match="CUDA"):
        B200LaserLstmEncoder(laser2_config(), {}, "cpu")
