"""Device-side timing of the top-k paths (CUDA events; not the bench contract): queries x 200k x 1472,
k = 100, every path that accepts the shape.  Writes gpurun_out/<tag>.json."""
import argparse, json, sys
from pathlib import Path
import torch
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from reprover_b200 import _native, synth
from reprover_b200.retrieval_ops import IndexHandle, sim_topk

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=200_000)
ap.add_argument("--d", type=int, default=1472)
ap.add_argument("--k", type=int, default=100)
ap.add_argument("--queries", default="1,2,3,4,5,8,16,64,128,256,1024")
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--tag", default="topk_bench")
ap.add_argument("--mask-frac", type=float, default=0.0, help="fraction of rows visible (contiguous runs); 0 = no mask")
args = ap.parse_args()
dev = torch.device("cuda:0")
E = synth.random_unit_rows(args.n, args.d, 1000, dev)
h = IndexHandle(E)
peak = 3350.0  # GB/s, HBM3 of the H100 SXM data sheet
out = {}
for nq in [int(x) for x in args.queries.split(",")]:
    Q = synth.random_unit_rows(nq, args.d, 999, dev)
    mask = None
    if args.mask_frac > 0:
        import numpy as np
        rng = np.random.default_rng(0)
        m = np.zeros((nq, (args.n + 31) // 32 * 32), dtype=bool)
        run = 4096
        for q in range(nq):
            starts = rng.choice(args.n // run, size=max(1, int(args.mask_frac * args.n / run)), replace=False)
            for s in starts:
                m[q, s * run:(s + 1) * run] = True
        m[:, args.n:] = False
        words = np.packbits(m.reshape(nq, -1, 8), axis=2, bitorder="little").reshape(nq, -1).view("<u4").copy()
        mask = torch.from_numpy(words.view(np.int32)).to(dev)
    for name, flags in (("auto", 0), ("mma", _native.RPX_TOPK_FORCE_MMA), ("stream", _native.RPX_TOPK_FORCE_STREAM)):
        if name == "stream" and nq > 2:
            continue
        for _ in range(5):
            sim_topk(Q, h, args.k, access_mask=mask, flags=flags)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        for _ in range(args.reps):
            sim_topk(Q, h, args.k, access_mask=mask, flags=flags)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        gbs = args.n * args.d * 2 / ms / 1e6
        rec = {"ms": ms, "qps": nq / ms * 1e3, "index_gbs": gbs, "hbm_frac": gbs / peak,
               "tflops": 2.0 * nq * args.n * args.d / ms / 1e9}
        out[f"q{nq}_{name}"] = rec
        print(nq, name, json.dumps(rec), flush=True)
out["stats"] = h.stats()
print("stats", out["stats"])
Path("gpurun_out").mkdir(exist_ok=True)
Path(f"gpurun_out/{args.tag}.json").write_text(json.dumps(out, indent=1))
