"""Time the fused image loss (bg_image_loss_fused: HWC4 render, 3 channels, the train step's weights and chain) at 1080p
and 4K with CUDA events, and compare builds of the library in one process.

  python scripts/loss_time.py [--lib A.so --lib B.so ...] [--rounds 5] [--iters 200] [--out result.json]

Each --lib is loaded side by side (ctypes, local symbols; each carries its own static CUDA runtime) and the builds are
timed in alternating rounds on the same inputs (each round one replay of a CUDA graph of --iters calls), so drift of the shared machine hits them alike.  Without --lib the
in-tree library is timed.  With two or more builds the script also reports whether their outputs (dL/dpred and the
per-block partials) are bit-identical on the same seeded inputs.  Prints one JSON line; --out also writes it to a file.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from brush_b200 import _lib  # noqa: E402

SIZES = [(1080, 1920), (2160, 3840)]


def _load(path: str):
    lib = C.CDLL(os.path.abspath(path))
    for name, (res, args) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    ctx = C.c_void_p()
    if lib.bg_ctx_create(0, 1024, 64, 64, 0, C.byref(ctx)) != 0:
        raise RuntimeError(f"bg_ctx_create failed for {path}")
    return lib, ctx


def _inputs(h, w, dev):
    rng = np.random.default_rng(h + w)
    pred = torch.from_numpy(rng.uniform(0, 1, (h, w, 4)).astype(np.float32)).to(dev)
    gt8 = rng.integers(0, 256, (h, w, 4), dtype=np.uint32)
    gt8[..., 3] = 255
    gt = (gt8[..., 0] | gt8[..., 1] << 8 | gt8[..., 2] << 16 | gt8[..., 3] << 24).astype(np.uint32)
    return pred, torch.from_numpy(gt.view(np.int32)).to(dev)


def _call(lib, ctx, pred, gt, out, part):
    h, w = pred.shape[0], pred.shape[1]
    npx = float(np.float32(w) * np.float32(h))
    chain = (C.c_float * 3)(*([float(np.float32(1.0) / np.float32(3.0 * npx))] * 3))
    st = lib.bg_image_loss_fused(ctx, torch.cuda.current_stream().cuda_stream, pred.data_ptr(), gt.data_ptr(), 3, h, w,
                                 1, w * 4, 4, 0.8, -0.2, None, 0, chain, out.data_ptr(), part.data_ptr())
    if st != 0:
        raise RuntimeError(f"bg_image_loss_fused returned {st}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loss_time.py needs a CUDA device")
    paths = args.lib or [_lib.LIB_PATH]
    libs = [_load(p) for p in paths]
    dev = torch.device("cuda", 0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    result = dict(gpu=q.stdout.strip() or torch.cuda.get_device_name(0), libs=paths, iters=args.iters, rounds=args.rounds,
                  sizes={})
    for h, w in SIZES:
        pred, gt = _inputs(h, w, dev)
        n_part = int(libs[0][0].bg_image_loss_num_partials(3, h, w))
        outs = [(torch.zeros_like(pred), torch.empty(n_part, dtype=torch.float32, device=dev)) for _ in libs]
        graphs = []
        for (lib, ctx), (o, p) in zip(libs, outs):
            for _ in range(10):
                _call(lib, ctx, pred, gt, o, p)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()   # device time only: the host's ctypes overhead stays out of the window
            with torch.cuda.graph(g):
                for _ in range(args.iters):
                    _call(lib, ctx, pred, gt, o, p)
            g.replay()
            graphs.append(g)
        torch.cuda.synchronize()
        times = [[] for _ in libs]
        for _ in range(args.rounds):
            for k, g in enumerate(graphs):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e3 / args.iters)
        entry = dict(us_per_call={p: dict(median=float(np.median(t)), min=float(min(t)), max=float(max(t)))
                                  for p, t in zip(paths, times)})
        if len(libs) > 1:
            entry["bit_identical"] = all(torch.equal(outs[0][0].view(torch.int32), o.view(torch.int32)) and
                                         torch.equal(outs[0][1].view(torch.int32), p.view(torch.int32)) for o, p in outs[1:])
        result["sizes"][f"{h}x{w}"] = entry
    for lib, ctx in libs:
        lib.bg_ctx_destroy(ctx)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
