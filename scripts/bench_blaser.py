"""Throughput of BLASER 2.0 scoring (``B200BlaserModel``, the card shapes: E = 1024, hidden [3072, 1536]) on one GPU, for
the reference-based (COMET, ``basic_ref``) and the quality-estimation (QE, ``basic_qe``) forms, against the reference's
own computation on the same card: ``F.normalize`` + ``torch.cat`` + ``nn.Sequential`` of Linear/Tanh on cuBLAS, in bf16
and in fp32, run in the same 65 536-pair passes as the engine.

Times 1 048 576 pairs (a mined corpus) and 64 pairs (latency); reports pairs/s, the achieved TFLOP/s from the FLOP count
of the shapes (2 (F 3072 + 3072 1536 + 1536) per pair, F = 6E or 4E) against NVIDIA's data-sheet dense bf16 rate of the
H100 SXM (989 TFLOP/s), the time of each kernel of one engine forward (torch.profiler, a separate untimed call), and the
agreement of the engine's scores with torch fp32 at 1 M pairs.  Device-timed with CUDA events; the card's name, power
limit and clocks are read in the same run.  Prints one JSON object (and writes it to ``--out`` if given).

    python scripts/bench_blaser.py [--steps 5] [--warmup 2] [--pairs 1048576] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

E, HIDDEN = 1024, [3072, 1536]
PASS = 65536
DATASHEET_BF16_TFLOPS = 989.0  # NVIDIA H100 SXM data sheet, dense bf16, 700 W


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


def flop_per_pair(form: str) -> int:
    f = (6 if form == "COMET" else 4) * E
    return 2 * (f * HIDDEN[0] + HIDDEN[0] * HIDDEN[1] + HIDDEN[1])


class TorchBlaser(torch.nn.Module):
    """The reference's forward (model.py:82-125) in eval mode, with torch modules in one dtype."""

    def __init__(self, form, sd, idx, dtype):
        super().__init__()
        self.form, self.dtype = form, dtype
        widths = [(6 if form == "COMET" else 4) * E] + HIDDEN + [1]
        layers = []
        for i in range(3):
            lin = torch.nn.Linear(widths[i], widths[i + 1])
            lin.load_state_dict({"weight": sd[f"mlp.{idx[i]}.weight"], "bias": sd[f"mlp.{idx[i]}.bias"]})
            layers += [lin, torch.nn.Tanh()] if i < 2 else [lin]
        self.mlp = torch.nn.Sequential(*layers).to(device="cuda", dtype=dtype)

    @torch.inference_mode()
    def forward(self, src, mt, ref, out):
        for i0 in range(0, src.shape[0], PASS):
            s, m = F.normalize(src[i0:i0 + PASS].to(self.dtype)), F.normalize(mt[i0:i0 + PASS].to(self.dtype))
            if self.form == "COMET":
                r = F.normalize(ref[i0:i0 + PASS].to(self.dtype))
                x = torch.cat([r, m, s * m, r * m, (m - s).abs(), (m - r).abs()], dim=-1)
            else:
                x = torch.cat([s, m, s * m, (m - s).abs()], dim=-1)
            out[i0:i0 + PASS] = self.mlp(x).float()
        return out


def _kernel_ms(fn) -> dict:
    """Device time per kernel of one call of fn(), from a torch.profiler trace (written to a temporary directory)."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ms = defaultdict(float)
    with tempfile.TemporaryDirectory() as d:
        trace = os.path.join(d, "blaser.pt.trace.json")
        prof.export_chrome_trace(trace)
        with open(trace) as f:
            events = json.load(f)["traceEvents"]
    for ev in events:
        if ev.get("cat") != "kernel":
            continue
        name = ev["name"]
        if "gemm_bf16_wgmma_kernel" in name:
            name = "gemm_hidden1_bf16_out" if "__nv_bfloat16" in name else "gemm_hidden2_fp32_out"
        elif "blaser_featurize_kernel" in name:
            name = "featurize"
        elif "blaser_output_kernel" in name:
            name = "output"
        ms[name] += ev["dur"] / 1e3  # us -> ms
    return dict(ms)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pairs", type=int, default=1 << 20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_blaser: no CUDA device (this measures the GPU engine)")
    torch.backends.cuda.matmul.allow_tf32 = False

    from oracle.blaser import make_synthetic_blaser_state_dict
    from sonar_b200 import B200BlaserModel, blaser_config, build
    from sonar_b200.blaser import linear_layer_indices

    build.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu": _gpu_info(), "pairs": args.pairs, "steps": args.steps, "datasheet_bf16_TFLOPs": DATASHEET_BF16_TFLOPS}
    n = args.pairs
    g = torch.Generator(device=dev).manual_seed(0)
    base = torch.randn(1, E, device=dev, generator=g)
    src, mt, ref = (base + 0.7 * torch.randn(n, E, device=dev, generator=g) for _ in range(3))
    for form, arch in (("COMET", "basic_ref"), ("QE", "basic_qe")):
        cfg = blaser_config(arch)
        sd = make_synthetic_blaser_state_dict(form, E, HIDDEN, cfg.dropout, seed=1)
        model = B200BlaserModel(cfg, sd, dev)
        idx = linear_layer_indices(cfg)
        tb = {"bf16": TorchBlaser(form, sd, idx, torch.bfloat16), "fp32": TorchBlaser(form, sd, idx, torch.float32)}
        r = ref if form == "COMET" else None
        out_t = torch.empty(n, 1, device=dev)
        row = {"flop_per_pair": flop_per_pair(form)}
        row["engine_ms"] = _time(lambda: model(src, mt, r), args.steps, args.warmup)
        for k, m in tb.items():
            row[f"torch_{k}_ms"] = _time(lambda: m(src, mt, ref, out_t), args.steps, args.warmup)
        for k in ("engine", "torch_bf16", "torch_fp32"):
            t = row[f"{k}_ms"] * 1e-3
            row[f"{k}_pairs_per_s"] = n / t
            row[f"{k}_TFLOPs"] = n * flop_per_pair(form) / t / 1e12
        row["engine_share_of_datasheet_bf16"] = row["engine_TFLOPs"] / DATASHEET_BF16_TFLOPS
        row["engine_speed_vs_torch_bf16"] = row["torch_bf16_ms"] / row["engine_ms"]
        row["engine_kernels_ms"] = _kernel_ms(lambda: model(src, mt, r))
        ks = row["engine_kernels_ms"]
        row["featurize_share_of_kernel_time"] = ks.get("featurize", 0.0) / max(sum(ks.values()), 1e-9)
        # latency: 64 pairs
        s64, m64, r64 = src[:64], mt[:64], ref[:64]
        out64 = torch.empty(64, 1, device=dev)
        row["latency_64_engine_ms"] = _time(lambda: model(s64, m64, r64 if r is not None else None), 50, 10)
        row["latency_64_torch_bf16_ms"] = _time(lambda: tb["bf16"](s64, m64, r64, out64), 50, 10)
        # agreement with torch fp32 at the timed size
        got = model(src, mt, r).double()
        want = tb["fp32"](src, mt, ref, out_t).double()
        d = (got - want).abs()
        std = float(want.std())
        pear = float(torch.corrcoef(torch.stack([got.flatten(), want.flatten()]))[0, 1])
        row["agreement_vs_torch_fp32"] = {"max_abs": float(d.max()), "mean_abs": float(d.mean()), "score_std": std,
                                          "pearson": pear,
                                          "ok": float(d.max()) <= 0.04 * std and float(d.mean()) <= 0.01 * std
                                          and pear >= 0.9995}
        bf = tb["bf16"](src, mt, ref, out_t).double()
        row["torch_bf16_vs_torch_fp32_max_abs"] = float((bf - want).abs().max())
        res[form] = row
        del model, tb
        torch.cuda.empty_cache()
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
