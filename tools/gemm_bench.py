"""Device-side timing (CUDA events) of the bare GEMM cores at the encoder's shapes for one 2^18-token call: rpx_gemm_bf16_f32 (128 x 256 throughput core) and cuBLAS."""
import json, sys
from pathlib import Path
import torch
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from reprover_b200 import _native

lib = _native.load()
dev = torch.device("cuda:0")
out = {}
for (M, N, K) in [(262144, 7168, 1472), (262144, 1472, 3584), (262144, 1152, 1472), (262144, 1472, 384)]:
    A = torch.randn(M, K, device=dev).to(torch.bfloat16)
    B = torch.randn(N, K, device=dev).to(torch.bfloat16)
    C = torch.empty(M, N, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    fn = lib.rpx_gemm_bf16_f32
    for _ in range(3):
        _native.check(fn(A.data_ptr(), B.data_ptr(), C.data_ptr(), M, N, K, st))
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn(A.data_ptr(), B.data_ptr(), C.data_ptr(), M, N, K, st)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    # cuBLAS reference point (library GEMM, not part of the product path)
    Cb = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    for _ in range(3):
        torch.matmul(A, B.t(), out=Cb)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        torch.matmul(A, B.t(), out=Cb)
    e1.record()
    torch.cuda.synchronize()
    ms_b = e0.elapsed_time(e1) / reps
    tf = 2.0 * M * N * K / ms / 1e9
    out[f"{M}x{N}x{K}"] = {"ms": ms, "tflops": tf, "cublas_ms": ms_b,
                           "cublas_tflops": 2.0 * M * N * K / ms_b / 1e9}
    print(M, N, K, f"{ms:.3f} ms  {tf:.1f} TF/s   cublas {ms_b:.3f} ms", flush=True)
Path("gpurun_out").mkdir(exist_ok=True)
Path("gpurun_out/gemm_bench.json").write_text(json.dumps(out, indent=1))
