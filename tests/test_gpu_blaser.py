"""BLASER 2.0 on the GPU: the GEMM's tanh epilogue, the featurize kernel, and the engine (``B200BlaserModel``) against the
reference module's golden, the float64 oracle at the card shapes, torch with the engine's rounding points, the reference's
behaviour, and bitwise batch-composition invariance."""

import math

import pytest
import torch
import torch.nn.functional as F

from oracle.blaser import OracleBlaser, make_blaser_inputs, make_synthetic_blaser_state_dict

pytestmark = pytest.mark.gpu

GOLDEN_PATH = "tests/golden/blaser_small.pt"
HIDDEN = [3072, 1536]
E = 1024


@pytest.fixture(scope="module")
def ops(native_lib, cuda_device):
    from sonar_b200 import ops as _ops

    torch.cuda.set_device(cuda_device)
    return _ops


def _rand(shape, scale, seed, device, dtype=torch.float32):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(device=device, dtype=dtype)


# the shapes of test_gpu_gemm_epilogues.py, and BLASER's second hidden layer at a batch tail
@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("m,n,k", [(1000, 1024, 1024), (4096, 2048, 256), (1000, 1536, 3072)])
def test_tanh_epilogue(ops, cuda_device, cta_group, m, n, k):
    a = _rand((m, k), 1.0, 41, cuda_device, torch.bfloat16)
    w = _rand((n, k), 1.0 / math.sqrt(k), 42, cuda_device, torch.bfloat16)
    bias = _rand((n,), 0.5, 43, cuda_device)
    y32 = ops.gemm_bf16(a, w, bias, epilogue="tanh", out_dtype=torch.float32, cta_group=cta_group)
    y16 = ops.gemm_bf16(a, w, bias, epilogue="tanh", cta_group=cta_group)
    assert torch.equal(y16, y32.to(torch.bfloat16))
    ref = torch.tanh(a.float() @ w.float().T + bias)
    torch.testing.assert_close(y32, ref, rtol=0, atol=2e-3)


def _inputs_on(device, n, e, seed=0):
    src, mt, ref = (t.to(device) for t in make_blaser_inputs(n, e, seed))
    for t in (src, mt, ref):
        t[n // 2] = 0.0  # a zero row
    return src, mt, ref


def _torch_features(src, mt, ref, form):
    if form == "COMET":
        return torch.cat([ref, mt, src * mt, ref * mt, torch.absolute(mt - src), torch.absolute(mt - ref)], dim=-1)
    return torch.cat([src, mt, src * mt, torch.absolute(mt - src)], dim=-1)


@pytest.mark.parametrize("form", ["COMET", "QE"])
@pytest.mark.parametrize("e", [32, 1024])
def test_featurize_kernel(ops, cuda_device, form, e):
    src, mt, ref = _inputs_on(cuda_device, 1000, e)
    # fp32 without normalisation: the same fp32 operations as torch.cat of the products and differences, so exact
    got = ops.blaser_featurize(src, mt, ref, form)
    assert torch.equal(got, _torch_features(src, mt, ref, form))
    # normalised: F.normalize sums the norm in another order, so a row's scale may differ in its last bit, and |mt - src|
    # cancels to small values that keep that absolute error (3e-8 measured); a zero row stays zero; bf16 = fp32 rounded
    n32 = ops.blaser_featurize(src, mt, ref, form, normalize=True)
    want = _torch_features(F.normalize(src), F.normalize(mt), F.normalize(ref), form)
    torch.testing.assert_close(n32, want, rtol=1e-6, atol=1e-7)
    assert bool(torch.isfinite(n32).all()) and float(n32[500].abs().max()) == 0.0
    n16 = ops.blaser_featurize(src, mt, ref, form, normalize=True, out_dtype=torch.bfloat16)
    assert torch.equal(n16, n32.to(torch.bfloat16))


def _model(cfg_kw, sd, device):
    from sonar_b200 import B200BlaserModel, blaser_config

    return B200BlaserModel(blaser_config("basic_ref", **cfg_kw), sd, device)


def test_engine_matches_the_reference_golden(native_lib, cuda_device):
    golden = torch.load(GOLDEN_PATH, weights_only=True)
    for c in golden["cases"]:
        model = _model(dict(input_form=c["input_form"], embedding_dim=c["embedding_dim"], hidden_dims=c["hidden_dims"],
                            dropout=c["dropout"]), c["state_dict"], cuda_device)
        out = model(c["src"], c["mt"], c["ref"]).cpu().double()
        want = c["out"]
        std = float(want.std())
        err = (out - want).abs()
        assert out.shape == (8, 1) and bool(torch.isfinite(out).all())
        assert float(err.max()) <= 0.04 * std, (c["input_form"], c["hidden_dims"], float(err.max()), std)
        feats = model.featurize_input(c["src"], c["mt"], c["ref"]).cpu().double()
        torch.testing.assert_close(feats, c["features"], rtol=1e-6, atol=1e-7)


@pytest.fixture(scope="module", params=["COMET", "QE"])
def card(request, native_lib, cuda_device):
    """(form, engine model, float64 oracle on the GPU, state dict) at the card shapes (E = 1024, [3072, 1536])."""
    form = request.param
    sd = make_synthetic_blaser_state_dict(form, E, HIDDEN, 0.1, seed=7 if form == "COMET" else 8)
    model = _model(dict(input_form=form), sd, cuda_device)
    oracle = OracleBlaser({k: v.to(cuda_device) for k, v in sd.items()}, input_form=form, hidden_dims=HIDDEN, dropout=0.1)
    return form, model, oracle, sd


def _scores(fn, src, mt, ref, form):
    return fn(src, mt, ref if form == "COMET" else None)


def test_engine_against_the_oracle(card, cuda_device):
    form, model, oracle, _ = card
    src, mt, ref = _inputs_on(cuda_device, 65537, E, seed=1)
    want = _scores(oracle, src, mt, ref, form).float()
    got = _scores(model, src, mt, ref, form)
    std = float(want[:4096].std())
    assert std > 0.3, std  # the recipe's spread (about 0.76)
    for n in (1, 10, 4096, 65537):  # the last one crosses the 65 536-row pass boundary
        g = model(src[:n], mt[:n], ref[:n]) if n < 65537 else got
        d = (g - want[:n]).abs()
        assert float(d.max()) <= 0.04 * std and float(d.mean()) <= 0.01 * std, (n, float(d.max()), float(d.mean()), std)
        if n >= 4096:
            r = torch.corrcoef(torch.stack([g.flatten().double(), want[:n].flatten().double()]))[0, 1]
            assert float(r) >= 0.9995, (n, float(r))


def test_engine_against_torch_with_the_engine_rounding(card, cuda_device):
    """torch in fp32 with the engine's rounding points: bf16 features, weights and first hidden layer; fp32 after."""
    form, model, _, sd = card
    src, mt, ref = _inputs_on(cuda_device, 65537, E, seed=2)
    from sonar_b200.blaser import blaser_config, linear_layer_indices

    idx = linear_layer_indices(blaser_config("basic_ref", input_form=form))
    w = [sd[f"mlp.{i}.weight"].to(cuda_device) for i in idx]
    b = [sd[f"mlp.{i}.bias"].to(cuda_device) for i in idx]
    x = _torch_features(F.normalize(src), F.normalize(mt), F.normalize(ref), form).to(torch.bfloat16).float()
    h1 = torch.tanh(x @ w[0].to(torch.bfloat16).float().T + b[0]).to(torch.bfloat16).float()
    h2 = torch.tanh(h1 @ w[1].to(torch.bfloat16).float().T + b[1])
    want = h2 @ w[2].T + b[2]
    got = _scores(model, src, mt, ref, form)
    d = (got - want).abs()
    assert float(d.max()) <= 5e-3 * float(want.std()), (float(d.max()), float(want.std()))


def test_reference_behaviour(card, cuda_device):
    form, model, _, _ = card
    src, mt, ref = _inputs_on(cuda_device, 10, E, seed=3)
    out = model(src, mt, ref)
    assert out.shape == (10, 1) and out.dtype == torch.float32 and out.device == cuda_device
    if form == "QE":
        assert torch.equal(model(src, mt), out)  # the reference is ignored
    else:
        with pytest.raises(ValueError, match="a reference embedding must be provided"):
            model(src, mt)
    # any float dtype, any device: cast to fp32 and moved
    half = [t.half().cpu() for t in (src, mt, ref)]
    assert torch.equal(model(*half), model(*[t.float().to(cuda_device) for t in half]))
    empty = torch.empty(0, E)
    assert model(empty, empty, empty).shape == (0, 1)
    with pytest.raises(ValueError, match="same N"):
        model(src, mt[:9], ref)
    with pytest.raises(ValueError, match="same N"):
        model(src[:, :512], mt[:, :512], ref[:, :512])


def test_batch_composition_invariance(card, cuda_device):
    """A pair's score has the same bits alone, inside a batch of 1000 and on both sides of the 65 536-row pass boundary."""
    form, model, _, _ = card
    src, mt, ref = _inputs_on(cuda_device, 66000, E, seed=4)
    pair = (src[:1], mt[:1], ref[:1])
    alone = model(*pair)
    for pos, n in ((517, 1000), (65535, 66000), (65536, 66000)):
        s, m, r = src[:n].clone(), mt[:n].clone(), ref[:n].clone()
        s[pos], m[pos], r[pos] = pair[0][0], pair[1][0], pair[2][0]
        assert torch.equal(model(s, m, r)[pos], alone[0]), (pos, n)
