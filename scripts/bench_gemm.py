"""Where the wgmma GEMM's time goes at the text encoder's shapes (M = 4096 x 128 tokens), on one GPU.

Default mode, one JSON line:
  * ``shapes``: the four GEMMs of an encoder layer through ``ops.gemm_bf16`` (``--cta-group``, default 2) -- QKV
    (N 3072, bias, bf16 out), out-projection (N 1024, fp32 ``x += ...``), FFN1 (N 8192, bias + ReLU, bf16 out), FFN2
    (N 1024, K 8192, fp32 ``x += ...``) -- and ``torch.nn.functional.linear`` in bf16 (cuBLAS) on the same operands
    as the yardstick for what this card reaches under its power limit.
  * ``k_sweep``: FFN1's M and N at K in {1024, 2048, 4096, 8192}, with the least-squares fit time = a + b K: ``a`` is the
    fixed cost per launch (the epilogues and pipeline fills of every tile), ``b`` the main-loop rate.
Device-timed with CUDA events over ``--iters`` launches after a warm-up; the card's name, power limit and SM clock are
read in the same call.  ``--cta-group 1`` runs independent CTAs instead of 2-CTA clusters that multicast the W tile.

``--profile DIR``: instead, one 4096 x 128 forward of the 24-layer encoder under ``torch.profiler`` (CUDA activities):
kernel time summed per kernel name as a share of the step, the trace written under DIR.

    python scripts/bench_gemm.py [--iters 10] [--cta-group {1,2}] [--out FILE]
    python scripts/bench_gemm.py --profile DIR
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

M, D, FFN = 4096 * 128, 1024, 8192
# name -> (N, K, ops.gemm_bf16 epilogue, fp32 accumulate output)
SHAPES = {"qkv": (3 * D, D, "bias", False), "out_proj": (D, D, "residual", True),
          "ffn1": (FFN, D, "relu", False), "ffn2": (D, FFN, "residual", True)}
SWEEP_K = (1024, 2048, 4096, 8192)


def _gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia_smi": (q, r.stdout.strip().splitlines()[0] if r.returncode == 0 else f"unavailable: {r.stderr.strip()}"),
            "torch_name": torch.cuda.get_device_name(0)}


def _time(fn, iters: int, warmup: int = 2) -> float:
    """Mean milliseconds of fn() between CUDA events over `iters` calls, after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / iters


def _operands(n: int, k: int, dev, seed: int):
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn((M, k), generator=g, device=dev).to(torch.bfloat16)
    w = (torch.randn((n, k), generator=g, device=dev) * k ** -0.5).to(torch.bfloat16)
    bias = torch.randn((n,), generator=g, device=dev) * 0.02
    return a, w, bias


def _shapes(ops, dev, iters: int, cta_group: int) -> dict:
    out = {}
    for i, (name, (n, k, epi, fp32)) in enumerate(SHAPES.items()):
        a, w, bias = _operands(n, k, dev, seed=i)
        c = torch.zeros((M, n), device=dev, dtype=torch.float32 if fp32 else torch.bfloat16)
        if fp32:  # x += a w^T + b in place: x grows a little per launch, the work does not change
            fn = lambda: ops.gemm_bf16(a, w, bias, epilogue=epi, residual=c, out=c, cta_group=cta_group)  # noqa: E731
        else:
            fn = lambda: ops.gemm_bf16(a, w, bias, epilogue=epi, out=c, cta_group=cta_group)  # noqa: E731
        flop = 2.0 * M * n * k
        ms = _time(fn, iters)
        ms_cublas = _time(lambda: torch.nn.functional.linear(a, w), iters)  # bf16 out, no epilogue
        out[name] = {"N": n, "K": k, "epilogue": epi + (" fp32 x +=" if fp32 else " bf16"),
                     "ms": ms, "TFLOPs": flop / ms / 1e9, "cublas_ms": ms_cublas, "cublas_TFLOPs": flop / ms_cublas / 1e9,
                     "vs_cublas": ms_cublas / ms}
        del a, w, bias, c
        torch.cuda.empty_cache()
    return out


def _k_sweep(ops, dev, iters: int, cta_group: int) -> dict:
    rows = []
    for k in SWEEP_K:
        a, w, bias = _operands(FFN, k, dev, seed=10 + k)
        c = torch.empty((M, FFN), device=dev, dtype=torch.bfloat16)
        ms = _time(lambda: ops.gemm_bf16(a, w, bias, epilogue="relu", out=c, cta_group=cta_group), iters)
        ms_cublas = _time(lambda: torch.nn.functional.linear(a, w), iters)
        rows.append({"K": k, "ms": ms, "TFLOPs": 2.0 * M * FFN * k / ms / 1e9, "cublas_ms": ms_cublas,
                     "cublas_TFLOPs": 2.0 * M * FFN * k / ms_cublas / 1e9})
        del a, w, bias, c
        torch.cuda.empty_cache()

    def fit(key):  # least squares time = a + b K
        ks = torch.tensor([float(r["K"]) for r in rows], dtype=torch.float64)
        ts = torch.tensor([r[key] for r in rows], dtype=torch.float64)
        kb, tb = ks.mean(), ts.mean()
        b = float(((ks - kb) * (ts - tb)).sum() / ((ks - kb) ** 2).sum())
        a = float(tb) - b * float(kb)
        return {"fixed_ms": a, "ms_per_1024_K": b * 1024,
                "main_loop_TFLOPs": 2.0 * M * FFN / (b * 1e-3) / 1e12}  # marginal rate of one more unit of K

    return {"M": M, "N": FFN, "rows": rows, "fit": fit("ms"), "fit_cublas": fit("cublas_ms")}


def _profile(out_dir: str, cta_group: int) -> dict:
    from torch.profiler import ProfilerActivity, profile

    import bench
    from sonar_b200 import B200TextEncoderModel, SequenceBatch, sonar_text_encoder_config

    dev = torch.device("cuda:0")
    model = B200TextEncoderModel(sonar_text_encoder_config("basic"), bench.synthetic_state_dict(dev), dev,
                                 cta_group=cta_group)
    g = torch.Generator().manual_seed(1000)
    batch = SequenceBatch(torch.randint(4, bench.VOCAB, (4096, 128), generator=g).to(dev), None)
    for _ in range(2):
        model(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model(batch)
        torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    trace = os.path.join(out_dir, "encoder_step.pt.trace.json")
    prof.export_chrome_trace(trace)
    per = {}
    with open(trace) as f:
        for ev in json.load(f)["traceEvents"]:
            if ev.get("cat") == "kernel":
                per[ev["name"]] = per.get(ev["name"], 0.0) + ev["dur"] / 1e3  # us -> ms
    total = sum(per.values())
    top = sorted(per.items(), key=lambda kv: -kv[1])
    kernels = [{"kernel": k[:160], "ms": v, "share": v / total} for k, v in top]
    gemm = sum(v for k, v in per.items() if "gemm_bf16_wgmma_kernel" in k)
    return {"kernel_ms_total": total, "gemm_wgmma_share": gemm / total, "kernels": kernels, "trace": trace}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--cta-group", type=int, default=2, choices=[1, 2])
    ap.add_argument("--profile", default="", metavar="DIR", help="profile one encoder step instead; trace under DIR")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm: no CUDA device (this measures the GPU kernels)")
    torch.backends.cuda.matmul.allow_tf32 = False

    from sonar_b200 import build, ops

    build.build()
    dev = torch.device("cuda:0")
    res = {"gpu": _gpu_info(), "M": M, "cta_group": args.cta_group}
    if args.profile:
        res["profile"] = _profile(args.profile, args.cta_group)
    else:
        res["shapes"] = _shapes(ops, dev, args.iters, args.cta_group)
        res["k_sweep"] = _k_sweep(ops, dev, args.iters, args.cta_group)
    res["gpu_after"] = _gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
