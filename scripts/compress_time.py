"""Timing of the compressed PLY export (development aid, not the bench): CUDA events around bg_compress_splats after
warm-up, and the whole export (device call, copy, file write) against the float export the training loop writes by
default, with the file sizes.  Random models generated on the device (K = 16 by default; the encoder's cost does not
depend on the values beyond the share of dropped rows, here none).  Prints one JSON line per size with the card and
its power limit.  Usage: compress_time.py [k] [n ...]"""
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import brush_b200.render as R
from brush_b200 import ply
from brush_b200.compress import compress_splats, splat_to_compressed_ply

k = int(sys.argv[1]) if len(sys.argv) > 1 else 16
sizes = [int(x) for x in sys.argv[2:]] or [1_000_000, 10_000_000]
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()


def model(n, dev):
    g = torch.Generator(device=dev).manual_seed(0xB2000510)
    u = lambda *s: torch.rand(*s, generator=g, device=dev)
    t = torch.cat([u(n, 3) * 20 - 10, u(n, 4) * 2 - 1, u(n, 3) * 4 - 7], 1)
    return t.contiguous(), (u(n, k, 3) - 0.5).contiguous(), (u(n) * 8 - 4).contiguous()


def float_export(t, sh, op, path):
    data = ply.splat_to_ply(t.cpu().numpy(), sh.cpu().numpy(), op.cpu().numpy())
    with open(path, "wb") as f:
        f.write(data)
    return len(data)


def compressed_export(ctx, t, sh, op, path):
    data = splat_to_compressed_ply(ctx, t, sh, op)
    with open(path, "wb") as f:
        f.write(data)
    return len(data)


for n in sizes:
    ctx = R.RenderContext(n, 16, 16)
    t, sh, op = model(n, ctx.device)
    for _ in range(3):                                     # warm-up
        enc = compress_splats(ctx, t, sh, op)
    torch.cuda.synchronize()
    reps = 20
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        compress_splats(ctx, t, sh, op)
    ev[1].record()
    torch.cuda.synchronize()
    kernel_ms = ev[0].elapsed_time(ev[1]) / reps
    m = int(enc.count.item())
    # the bytes the encoding needs: every source row read once, the m encoded rows and the chunk rows written
    need = n * (44 + 12 * k) + m * (16 + 3 * (k - 1)) + 72 * ((m + 255) // 256)
    # what this implementation moves besides: the second (gathered) read of the kept rows, the means for the keys,
    # keys / indices through four sort passes, the order read and written
    moved = need + m * (44 + 12 * k) + n * (12 + 8 + 4) + 4 * n * 16 + 8 * m
    with tempfile.TemporaryDirectory() as d:
        rec = {"n": n, "k": k, "m": m, "compress_ms": kernel_ms, "bytes_needed": need,
               "needed_GBps": need / kernel_ms / 1e6, "bytes_moved_est": moved, "moved_GBps": moved / kernel_ms / 1e6}
        for name, fn in (("float", lambda p: float_export(t, sh, op, p)), ("compressed", lambda p: compressed_export(ctx, t, sh, op, p))):
            fn(os.path.join(d, "warm.ply"))
            times = []
            for i in range(3 if n <= 2_000_000 else 1):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                size = fn(os.path.join(d, f"{name}_{i}.ply"))
                times.append(time.perf_counter() - t0)
                os.remove(os.path.join(d, f"{name}_{i}.ply"))
            rec[f"{name}_export_s"] = min(times)
            rec[f"{name}_bytes"] = size
            rec[f"{name}_bytes_per_splat"] = size / n
        rec["card"] = smi
        print(json.dumps(rec), flush=True)
    del t, sh, op, enc
    ctx.close()
    torch.cuda.empty_cache()
