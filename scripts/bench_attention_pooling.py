"""Cost of the text encoder's attention pooler (``pooling="attention"``) on one GPU.

Times the `basic` encoder (24 layers, D = 1024) with MEAN pooling and with the 24-layer attention pooler (E = 1024, 16
heads) at 4096 x 128 tokens and on ragged lengths U{16..128}, the latent cross-attention kernel alone (achieved
bandwidth against the T * D * 2 bytes of memory it must read per pooler layer), and the device memory the handle
allocates for the absorbed weights.  Device-timed with CUDA events; the card's name, power limit and clocks are read
in the same run.  Prints one JSON object (and writes it to ``--out`` if given).

    python scripts/bench_attention_pooling.py [--steps 5] [--warmup 2] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VOCAB = 32000  # the embedding lookup reads one row per token whatever the vocabulary size


def _gpu_info() -> dict:
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia_smi": r.stdout.strip().splitlines()[0] if r.returncode == 0 else f"unavailable: {r.stderr.strip()}",
            "torch_name": torch.cuda.get_device_name(0)}


def _time(fn, steps: int, warmup: int) -> float:
    """Mean milliseconds of fn() between CUDA events over `steps` calls, after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / steps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--seq-len", type=int, default=128)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention_pooling: no CUDA device (this measures the GPU engine)")

    from oracle.text_attention_pooler import OracleAttentionEncoderConfig, make_synthetic_attention_state_dict
    from sonar_b200 import (B200TextEncoderModel, PaddingMask, SequenceBatch, VocabularyInfo, build, ops,
                            sonar_text_encoder_config)

    build.build()
    dev = torch.device("cuda:0")
    res = {"gpu": _gpu_info(), "batch": args.batch, "seq_len": args.seq_len, "steps": args.steps}
    sd = make_synthetic_attention_state_dict(OracleAttentionEncoderConfig(vocab_size=VOCAB), seed=1)
    vocab = VocabularyInfo(size=VOCAB, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1)
    mean = B200TextEncoderModel(sonar_text_encoder_config("basic", vocab_info=vocab), sd, dev)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    attn = B200TextEncoderModel(sonar_text_encoder_config("basic", vocab_info=vocab, pooling="attention"), sd, dev)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info(dev)[0]
    del sd
    d, hd, layers = 1024, 16, 24
    res["handle_extra_bytes_formula"] = layers * (2 * hd * d * d * 2 + (hd * d + d) * 4)
    # the attention model's own weight copies (pooler matrices, ~ 24 * 24M bf16 parameters) are included here
    res["create_device_bytes_measured"] = free0 - free1

    b, s = args.batch, args.seq_len
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(4, VOCAB, (b, s), generator=g).to(dev)
    ragged = torch.randint(16, s + 1, (b,), generator=g).tolist()
    for name, lens in (("dense", [s] * b), ("ragged_16_128", ragged)):
        batch = SequenceBatch(ids, PaddingMask(torch.tensor(lens), s, lens))
        t_mean = _time(lambda: mean(batch), args.steps, args.warmup)
        t_attn = _time(lambda: attn(batch), args.steps, args.warmup)
        res[name] = {"tokens": sum(lens), "mean_pool_ms": t_mean, "attention_pool_ms": t_attn,
                     "pooler_added_ms": t_attn - t_mean, "pooler_share_of_step": (t_attn - t_mean) / t_attn}

    # the latent kernel alone, at the dense shape
    t_tok = b * s
    mem = torch.randn(t_tok, d, device=dev).to(torch.bfloat16)
    qt = (torch.randn(b, hd, d, device=dev) * 0.05).to(torch.bfloat16)
    cu = ops.cu_seqlens_of([s] * b).to(dev)
    t_k = _time(lambda: ops.pool_latent_attention(qt, mem, cu), 20, 3)
    need = t_tok * d * 2
    res["latent_kernel"] = {"ms": t_k, "memory_bytes": need, "achieved_GBps": need / (t_k * 1e-3) / 1e9,
                            "share_of_3350_GBps": need / (t_k * 1e-3) / 3.35e12, "per_step_24_layers_ms": 24 * t_k}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
