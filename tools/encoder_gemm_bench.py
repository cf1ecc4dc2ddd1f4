"""Device-side timing (CUDA events) of the encoder's four GEMMs (QKV, O-proj, FFN-up, FFN-down), launched as the
throughput path launches them (rpx_debug_encoder_gemm), at one 2^18-token call of ByT5-small (d_model 1472,
6 heads, d_ff 3584).  O-proj is memory-bound: its achieved bandwidth counts the bytes one token must move
(attn in, h32 read and written, h16 out, the RMSNorm partial sums out).

    python tools/encoder_gemm_bench.py [--tokens T] [--reps R] [--sites qkv,oproj,ffn_up,ffn_down] [--out FILE]
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
# site -> (id, N, K); A is [T, K], B is [N, K]
SITES = {
    "qkv": (_native.RPX_EGEMM_QKV, 3 * INNER, D),
    "oproj": (_native.RPX_EGEMM_OPROJ, D, INNER),
    "ffn_up": (_native.RPX_EGEMM_FFN_UP, 2 * F, D),
    "ffn_down": (_native.RPX_EGEMM_FFN_DOWN, D, F),
}
RESIDUAL = ("oproj", "ffn_down")


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
    ap.add_argument("--sites", default=",".join(SITES), help="comma-separated subset of " + ", ".join(SITES))
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    sites = args.sites.split(",")
    unknown = [s for s in sites if s not in SITES]
    if unknown:
        sys.exit(f"encoder_gemm_bench: unknown site(s) {unknown}")
    if not torch.cuda.is_available():
        sys.exit("encoder_gemm_bench: no CUDA device")
    lib = _native.load()
    dev = torch.device("cuda:0")
    T = args.tokens
    g = torch.Generator(device=dev).manual_seed(0)
    parts = math.ceil(D / 128)
    h32 = torch.randn(T, D, generator=g, device=dev)
    h16 = torch.empty(T, D, dtype=torch.bfloat16, device=dev)
    ss = torch.empty(parts * T, device=dev)
    # RMSNorm partial sums of the gated sites' input: positive, about d_model / parts per part
    ss_in = torch.rand(parts * T, generator=g, device=dev) * (2 * D / parts)
    st = torch.cuda.current_stream().cuda_stream
    result = {"tokens": T, "reps": args.reps, "library": _native.library_path().name}
    for site in sites:
        sid, N, K = SITES[site]
        A = torch.randn(T, K, generator=g, device=dev).to(torch.bfloat16)
        B = (torch.randn(N, K, generator=g, device=dev) / math.sqrt(K)).to(torch.bfloat16)
        if site in RESIDUAL:
            def call():
                return lib.rpx_debug_encoder_gemm(sid, 0, A.data_ptr(), B.data_ptr(), T, N, K, 1e-6, None, None,
                                                  h32.data_ptr(), h16.data_ptr(), ss.data_ptr(), None, 0, st)
        else:
            out = torch.empty(T, N // 2 if site == "ffn_up" else N, dtype=torch.bfloat16, device=dev)

            def call():
                return lib.rpx_debug_encoder_gemm(sid, 0, A.data_ptr(), B.data_ptr(), T, N, K, 1e-6, ss_in.data_ptr(),
                                                  out.data_ptr(), None, None, None, None, 0, st)

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
        r = {"ms": ms, "tflops": 2.0 * T * N * K / ms / 1e9}
        line = f"{site:9s} T={T} N={N} K={K}: {ms:.3f} ms  {r['tflops']:.1f} TFLOP/s"
        if site == "oproj":
            r["bytes_per_token"] = token_bytes(K)
            r["hbm_tb_per_s"] = T * token_bytes(K) / ms / 1e9
            line += f"  {r['hbm_tb_per_s']:.2f} TB/s over {r['bytes_per_token']} B/token"
        result[site] = r
        print(line, flush=True)
        del A, B, call
        if site not in RESIDUAL:
            del out
    result["gpu"] = board()
    print(json.dumps(result))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
