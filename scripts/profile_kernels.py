"""Small driver for profiler captures (Nsight Compute, or torch.profiler around it): runs each hot kernel a few times at
the bench shapes.
    ncu --set full --clock-control none --import-source on -k regex:gemm_bf16 -s 2 -c 2 -o gemm python scripts/profile_kernels.py gemm
"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sonar_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
which = sys.argv[1] if len(sys.argv) > 1 else "gemm"
T, D, F = 4096 * 128, 1024, 8192
if len(sys.argv) > 2:
    T = int(sys.argv[2])
g = torch.Generator(device=dev).manual_seed(0)
if which == "gemm":      # FFN inner projection (bias + ReLU, bf16 out)
    a = torch.randn((T, D), device=dev, generator=g).to(torch.bfloat16)
    w = (torch.randn((F, D), device=dev, generator=g) / math.sqrt(D)).to(torch.bfloat16)
    b = torch.randn((F,), device=dev, generator=g)
    out = torch.empty((T, F), device=dev, dtype=torch.bfloat16)
    for _ in range(4):
        ops.gemm_bf16(a, w, b, epilogue="relu", out=out)
elif which == "gemm_res":  # out-proj (bias + fp32 residual in place)
    a = torch.randn((T, D), device=dev, generator=g).to(torch.bfloat16)
    w = (torch.randn((D, D), device=dev, generator=g) / math.sqrt(D)).to(torch.bfloat16)
    b = torch.randn((D,), device=dev, generator=g)
    x = torch.randn((T, D), device=dev, generator=g)
    for _ in range(4):
        ops.gemm_bf16(a, w, b, epilogue="residual", residual=x, out=x)
elif which == "gemm_resstats":  # out-proj with the LayerNorm-folding producer epilogue (x += ..., bf16 copy, row statistics)
    a = torch.randn((T, D), device=dev, generator=g).to(torch.bfloat16)
    w = (torch.randn((D, D), device=dev, generator=g) / math.sqrt(D)).to(torch.bfloat16)
    b = torch.randn((D,), device=dev, generator=g)
    x = torch.randn((T, D), device=dev, generator=g)
    for _ in range(4):
        ops.gemm_residual_stats(a, w, b, x)
elif which == "attention":
    qkv = torch.randn((T, 3 * D), device=dev, generator=g).to(torch.bfloat16)
    cu = ops.cu_seqlens_of([128] * (T // 128)).to(dev)
    for _ in range(4):
        ops.attention(qkv, cu, 16)
elif which == "layernorm":
    x = torch.randn((T, D), device=dev, generator=g)
    gg, bb = torch.ones(D, device=dev), torch.zeros(D, device=dev)
    for _ in range(4):
        ops.layernorm(x, gg, bb)
elif which == "fbank":   # 256 x 10 s waveforms -> 80-bin fbank + standardise (BASELINE config 3 frontend)
    from sonar_b200.speech_frontend import WaveformToFbank
    conv = WaveformToFbank(dev)
    waves = [(torch.randn(160000, device=dev, generator=g) * 0.05).clamp(-1, 1) for _ in range(256)]
    for _ in range(3):
        conv(waves)
elif which == "xsim":    # k-NN of 65536 x 65536 (normalise, wgmma GEMM + running top-16, fp64 re-rank)
    from sonar_b200 import xsim
    y = torch.randn((65536, 1024), device=dev, generator=g)
    x = y + 0.1 * torch.randn((65536, 1024), device=dev, generator=g)
    for _ in range(3):
        xsim.knn(x, y, 4)
elif which == "speech":  # one full speech-encoder forward (64 x 10 s), for a launch list
    from oracle.speech_encoder import OracleSpeechConfig, make_synthetic_speech_state_dict
    from sonar_b200 import B200SpeechEncoderModel, PaddingMask, SequenceBatch, sonar_speech_encoder_config
    sd = make_synthetic_speech_state_dict(OracleSpeechConfig(), seed=3)
    model = B200SpeechEncoderModel(sonar_speech_encoder_config("english"), sd, dev)
    fb = torch.randn((64, 998, 80), device=dev)
    fr = [998] * 64
    for _ in range(2):
        model(SequenceBatch(fb, PaddingMask(torch.tensor(fr), 998, fr)))
elif which in ("decoder", "decoder_small"):  # a few decoder steps (512 x beam 5, or the pipelines' default 5 x beam 5)
    from sonar_b200 import B200TextDecoderModel, sonar_text_decoder_config
    gg = torch.Generator(device=dev).manual_seed(3)
    sd = {}
    def rn(*shape, s=0.02):
        return torch.randn(*shape, generator=gg, device=dev) * s
    sd["decoder_frontend.embed.weight"] = rn(256206, 1024, s=1 / 32)
    for i in range(24):
        p = f"decoder.layers.{i}."
        for a in ("self_attn", "encoder_decoder_attn"):
            for nme in ("q_proj", "k_proj", "v_proj", "output_proj"):
                sd[p + f"{a}.{nme}.weight"], sd[p + f"{a}.{nme}.bias"] = rn(1024, 1024), rn(1024)
            sd[p + f"{a}_layer_norm.weight"], sd[p + f"{a}_layer_norm.bias"] = 1 + rn(1024), rn(1024)
        sd[p + "ffn.inner_proj.weight"], sd[p + "ffn.inner_proj.bias"] = rn(8192, 1024), rn(8192)
        sd[p + "ffn.output_proj.weight"], sd[p + "ffn.output_proj.bias"] = rn(1024, 8192), rn(1024)
        sd[p + "ffn_layer_norm.weight"], sd[p + "ffn_layer_norm.bias"] = 1 + rn(1024), rn(1024)
    sd["decoder.layer_norm.weight"], sd["decoder.layer_norm.bias"] = 1 + rn(1024), rn(1024)
    model = B200TextDecoderModel(sonar_text_decoder_config("basic"), sd, dev)
    n, beam, tmax = (512 if which == "decoder" else 5), 5, 130
    model.begin(torch.randn((n, 1024), device=dev) * 0.25, beam, tmax)
    r = n * beam
    table = torch.arange(r, dtype=torch.int32, device=dev)[:, None].expand(r, tmax).contiguous()
    tk = torch.randint(4, 256000, (r,), device=dev)
    for t in (0, 1, 64, 120):
        model.step(tk, table, t)
elif which == "text_step":  # three forwards of the benched text encoder (4096 x 128): 170 kernels per forward
    from bench import BATCH, SEQ, VOCAB, synthetic_state_dict
    from sonar_b200 import B200TextEncoderModel, SequenceBatch, sonar_text_encoder_config
    model = B200TextEncoderModel(sonar_text_encoder_config("basic"), synthetic_state_dict(dev), dev)
    ids = torch.randint(4, VOCAB, (BATCH, SEQ), device=dev, dtype=torch.int64)
    for _ in range(3):
        model(SequenceBatch(ids, None))
elif which == "xsim_bidir":  # both k-NN directions from one sweep, at the bench size (config 5)
    from sonar_b200 import xsim
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 262144
    y = torch.randn((n, 1024), device=dev, generator=g)
    x = y + 0.1 * torch.randn((n, 1024), device=dev, generator=g)
    for _ in range(2):
        xsim.knn_bidir(x, y, 4)
torch.cuda.synchronize()
print("done", which)
