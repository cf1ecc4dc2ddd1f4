"""Device-side timing (CUDA events) of the encoder's two residual GEMMs, O-proj and FFN-down, launched as the
throughput path launches them (rpx_debug_encoder_gemm), at one 2^18-token call of ByT5-small (d_model 1472,
6 heads, d_ff 3584).  O-proj is memory-bound: its achieved bandwidth counts the bytes one token must move
(attn in, h32 read and written, h16 out, the RMSNorm partial sums out).

    python tools/residual_gemm_bench.py [--tokens T] [--reps R] [--out FILE]
"""
import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from reprover_b200 import _native  # noqa: E402

D, INNER, F = 1472, 6 * 64, 3584
SITES = {"oproj": (_native.RPX_EGEMM_OPROJ, INNER), "ffn_down": (_native.RPX_EGEMM_FFN_DOWN, F)}


def board():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, check=True)
        name, power, clock = (s.strip() for s in out.stdout.strip().split(","))
        return {"name": name, "power_limit_w": float(power), "sm_clock_mhz_after": float(clock)}
    except (OSError, subprocess.CalledProcessError, ValueError):
        return {"name": torch.cuda.get_device_name(), "power_limit_w": None, "sm_clock_mhz_after": None}


def token_bytes(K):
    """HBM bytes per token of a residual GEMM: A row (bf16), h32 read + write, h16 write, one fp32 partial sum
    per 128 columns.  The weights stay in L2."""
    return 2 * K + 2 * 4 * D + 2 * D + 4 * math.ceil(D / 128)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=1 << 18)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("residual_gemm_bench: no CUDA device")
    lib = _native.load()
    dev = torch.device("cuda:0")
    T = args.tokens
    g = torch.Generator(device=dev).manual_seed(0)
    h32 = torch.randn(T, D, generator=g, device=dev)
    h16 = torch.empty(T, D, dtype=torch.bfloat16, device=dev)
    ss = torch.empty(math.ceil(D / 128) * T, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    result = {"tokens": T, "reps": args.reps}
    for site, (sid, K) in SITES.items():
        A = torch.randn(T, K, generator=g, device=dev).to(torch.bfloat16)
        B = (torch.randn(D, K, generator=g, device=dev) / math.sqrt(K)).to(torch.bfloat16)

        def call():
            return lib.rpx_debug_encoder_gemm(sid, 0, A.data_ptr(), B.data_ptr(), T, D, K, 1e-6, None, None,
                                              h32.data_ptr(), h16.data_ptr(), ss.data_ptr(), None, 0, st)

        for _ in range(3):
            _native.check(call())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            call()
        e1.record()
        torch.cuda.synchronize()
        _native.check(call())
        ms = e0.elapsed_time(e1) / args.reps
        r = {"ms": ms, "tflops": 2.0 * T * D * K / ms / 1e9, "hbm_tb_per_s": T * token_bytes(K) / ms / 1e9,
             "bytes_per_token": token_bytes(K)}
        result[site] = r
        print(f"{site:9s} T={T} K={K}: {ms:.3f} ms  {r['tflops']:.1f} TFLOP/s  "
              f"{r['hbm_tb_per_s']:.2f} TB/s over {r['bytes_per_token']} B/token", flush=True)
        del A, B
    result["gpu"] = board()
    print(json.dumps(result))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
