"""BASELINE config 5: encoder throughput sweep seq_len {128,512,1024,2048} x batch {32,128,512} on 1 H100,
roofline fraction.  ids ~ UniformInt[3,258], full-length masks (SURVEY 8d), through `_encode`-equivalent
packed calls (rpx_encode_bytes with fixed-length strings; EOS included in seq_len).  CUDA events, 3 warm-ups."""
import json, sys
from pathlib import Path
import numpy as np, torch
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from reprover_b200 import synth
from reprover_b200.engine import T5EncoderEngine

dev = torch.device("cuda:0")
peaks = {"bf16_tflops_sustained": 989.0, "bf16_tflops": 989.0}  # H100 SXM data sheet, dense bf16
cfg = dict(synth.BYT5_SMALL)
eng = T5EncoderEngine(cfg, synth.random_t5_state_dict(cfg, seed=synth.SEED), dev, max_tokens_per_call=1 << 18)
rows = []
rng = np.random.default_rng(synth.SEED)
for L in (128, 512, 1024, 2048):
    for B in (32, 128, 512):
        data = rng.integers(0, 256, size=B * (L - 1), dtype=np.uint8)   # ids 3..258 = bytes 0..255
        offsets = np.arange(B + 1, dtype=np.int64) * (L - 1)
        d = torch.from_numpy(data).to(dev)
        out = torch.empty(B, 1472, dtype=torch.bfloat16, device=dev)
        per_call = max(1, (1 << 18) // L)
        def step():
            for a in range(0, B, per_call):
                b = min(B, a + per_call)
                eng.encode_packed_bytes(d[offsets[a]:offsets[b]], offsets[a:b + 1] - offsets[a], L, out[a:b])
        for _ in range(3): step()
        reps = max(3, int(2e5 // (B * L)) )
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        for _ in range(reps): step()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        flops = B * L * (434_110_464.0 + 18_432.0 * L)
        tf = flops / ms / 1e9
        rows.append({"seq_len": L, "batch": B, "tokens": B * L, "ms": ms, "seq_per_s": B / ms * 1e3, "tflops": tf,
                     "frac_of_sustained_peak": tf / peaks["bf16_tflops_sustained"], "frac_of_burst_peak": tf / peaks["bf16_tflops"]})
        print(rows[-1], flush=True)
Path("gpurun_out").mkdir(exist_ok=True)
Path("gpurun_out/sweep_encoder.json").write_text(json.dumps({"peaks": peaks, "rows": rows}, indent=1))
