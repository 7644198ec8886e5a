"""Throughput of the LASER2 text encoder (``B200LaserLstmEncoder``, the `laser2` shape: vocab 50004, 320 -> 5 x
bidirectional LSTM 512, max over time) on one GPU, against the reference's own computation on the same card:
``torch.nn.LSTM`` over ``pack_padded_sequence`` + ``pad_packed_sequence`` + the masked max (cuDNN), in bf16 and in fp32.

Times 4096 x 128 tokens and ragged lengths U{16..128}; the recurrent kernel alone per layer and the input GEMMs alone
(achieved FLOP/s and bytes/s from the arithmetic of the shapes); checks the engine on a 256-sentence subset against the
float64 oracle.  Device-timed with CUDA events; the card's name, power limit and clocks are read in the same run.
Prints one JSON object (and writes it to ``--out`` if given).

    python scripts/bench_laser2.py [--steps 5] [--warmup 2] [--out FILE]
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

H, E, LAYERS, DIRS, VOCAB, PAD = 512, 320, 5, 2, 50004, 1
WEIGHT_BOUND = 0.1  # see tests/test_gpu_laser2.py: keeps sentence embeddings apart


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


class CudnnLaser2(torch.nn.Module):
    """The reference model's computation with torch modules: embedding, length sort, packed nn.LSTM (cuDNN on CUDA),
    pad_packed_sequence(0.0), positions holding pad_idx set to -inf, max over time, unsort."""

    def __init__(self, sd, dtype):
        super().__init__()
        self.embed = torch.nn.Embedding(VOCAB, E, padding_idx=PAD)
        self.lstm = torch.nn.LSTM(E, H, num_layers=LAYERS, bidirectional=True)
        self.embed.load_state_dict({"weight": sd["embed_tokens.weight"]})
        self.lstm.load_state_dict({k[len("lstm."):]: v for k, v in sd.items() if k.startswith("lstm.")})
        self.to(device="cuda", dtype=dtype)

    @torch.inference_mode()
    def forward(self, seqs, lens):
        order = torch.argsort(-lens)
        x = self.embed(seqs[order]).transpose(0, 1)
        packed = torch.nn.utils.rnn.pack_padded_sequence(x, lens[order].cpu())
        out, _ = self.lstm(packed)
        y, _ = torch.nn.utils.rnn.pad_packed_sequence(out, padding_value=0.0)
        y = y.float().masked_fill_(seqs[order].eq(PAD).t().unsqueeze(-1), float("-inf"))
        return y.max(dim=0).values[torch.argsort(order)]


def _flops_bytes(tokens: int) -> dict:
    """Arithmetic of the shapes: input GEMMs 2 * T * 4H * in * dirs per layer, recurrences 2 * T * 4H * H * dirs per layer;
    G (bf16) written and read once per layer."""
    gemm = sum(2 * tokens * 4 * H * (E if l == 0 else DIRS * H) * DIRS for l in range(LAYERS))
    rec = LAYERS * 2 * tokens * 4 * H * H * DIRS
    g_bytes = LAYERS * 2 * tokens * DIRS * 4 * H * 2
    return {"gemm_flop": gemm, "recurrent_flop": rec, "g_bytes": g_bytes}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--seq-len", type=int, default=128)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_laser2: no CUDA device (this measures the GPU engine)")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    from oracle.laser_lstm import OracleLaser2, OracleLaser2Config, make_synthetic_laser2_state_dict
    from sonar_b200 import B200LaserLstmEncoder, build, laser2_config, ops

    build.build()
    dev = torch.device("cuda:0")
    res = {"gpu": _gpu_info(), "batch": args.batch, "seq_len": args.seq_len, "steps": args.steps}
    ocfg = OracleLaser2Config()
    sd = make_synthetic_laser2_state_dict(ocfg, seed=1, weight_bound=WEIGHT_BOUND)
    model = B200LaserLstmEncoder(laser2_config(), sd, dev)
    cudnn = {"bf16": CudnnLaser2(sd, torch.bfloat16), "fp32": CudnnLaser2(sd, torch.float32)}

    b, s = args.batch, args.seq_len
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(3, VOCAB, (b, s), generator=g)
    ragged = torch.randint(16, s + 1, (b,), generator=g)
    ragged[0] = s  # the padded width equals the longest sentence, as the reference requires
    for name, lens in (("dense", torch.full((b,), s)), ("ragged_16_128", ragged)):
        ids_l = ids.clone()
        ids_l[torch.arange(s)[None, :] >= lens[:, None]] = PAD
        d_ids, d_lens = ids_l.to(dev), lens.to(dev)
        tokens = int(lens.sum())
        row = {"tokens": tokens}
        row["engine_ms"] = _time(lambda: model(d_ids, lens), args.steps, args.warmup)
        for k, m in cudnn.items():
            try:
                row[f"cudnn_{k}_ms"] = _time(lambda: m(d_ids, d_lens), args.steps, args.warmup)
            except RuntimeError as e:  # reported, not hidden: the comparison is then missing from the result
                row[f"cudnn_{k}_error"] = str(e)[:300]
        for k in ("engine", "cudnn_bf16", "cudnn_fp32"):
            if f"{k}_ms" in row:
                row[f"{k}_sentences_per_s"] = b / (row[f"{k}_ms"] * 1e-3)
        fb = _flops_bytes(tokens)
        row["engine_achieved_TFLOPs"] = (fb["gemm_flop"] + fb["recurrent_flop"]) / (row["engine_ms"] * 1e-3) / 1e12
        if "cudnn_bf16_ms" in row:
            row["speedup_vs_cudnn_bf16"] = row["cudnn_bf16_ms"] / row["engine_ms"]
        res[name] = row

    # the two halves of a layer alone, at the dense shape (layer 1..4 input width 1024)
    T = b * s
    x = (torch.randn(T, DIRS * H, device=dev) * 0.5).bfloat16()
    w_ih = ((torch.rand(DIRS * 4 * H, DIRS * H, device=dev) * 2 - 1) * WEIGHT_BOUND).bfloat16()
    bias = torch.zeros(DIRS * 4 * H, device=dev)
    gbuf = torch.empty(T, DIRS * 4 * H, device=dev, dtype=torch.bfloat16)
    t_gemm = _time(lambda: ops.gemm_bf16(x, w_ih, bias, out=gbuf), 10, 2)
    w_hh = ((torch.rand(DIRS * 4 * H, H, device=dev) * 2 - 1) * WEIGHT_BOUND).bfloat16()
    cu = ops.cu_seqlens_of([s] * b).to(dev)
    tiles = torch.arange(((b + 63) // 64) * 64, dtype=torch.int32)
    tiles[tiles >= b] = -1
    tiles = tiles.to(dev)
    t_rec = _time(lambda: ops.lstm_recurrent(gbuf, w_hh, cu, tiles, DIRS), 5, 1)
    gemm_flop = 2 * T * DIRS * 4 * H * DIRS * H
    rec_flop = 2 * T * 4 * H * H * DIRS
    res["layer_1024_in"] = {
        "input_gemm_ms": t_gemm, "input_gemm_TFLOPs": gemm_flop / (t_gemm * 1e-3) / 1e12,
        "recurrent_ms": t_rec, "recurrent_TFLOPs": rec_flop / (t_rec * 1e-3) / 1e12,
        "recurrent_us_per_time_step_of_the_batch": t_rec * 1e3 / s,
        "g_bytes_per_layer": T * DIRS * 4 * H * 2, "g_write_read_GBps_at_gemm_plus_rec":
            2 * T * DIRS * 4 * H * 2 / ((t_gemm + t_rec) * 1e-3) / 1e9,
    }

    # accuracy on a 256-sentence subset of the ragged batch against the float64 oracle
    n = 256
    sub_lens = ragged[:n]
    sub = ids[:n, : int(sub_lens.max())].clone()
    sub[torch.arange(sub.shape[1])[None, :] >= sub_lens[:, None]] = PAD
    got = model(sub.to(dev), sub_lens).double().cpu()
    ref = OracleLaser2(ocfg, sd, dtype=torch.float64, device=dev)(sub, sub_lens).cpu()
    cos = torch.nn.functional.cosine_similarity(got, ref, dim=1)
    mu = ref.mean(0, keepdim=True)
    res["accuracy_256"] = {"one_minus_cos_max": float((1 - cos).max()),
                           "centred_cos_min": float(torch.nn.functional.cosine_similarity(got - mu, ref - mu, dim=1).min()),
                           "rel_l2_max": float(((got - ref).norm(dim=1) / ref.norm(dim=1)).max())}
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
