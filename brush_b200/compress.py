"""SuperSplat compressed PLY export over the C ABI (the reference reads this layout, import.rs:408-600, but never
writes it).

  compress_splats          <- bg_compress_splats: validity, Morton order, per-chunk ranges and quantisation on the
                              device (DESIGN.md section 4.8); the encoding stays on the device
  splat_to_compressed_ply  <- the file: one call, one readback of the kept count, a copy of the m encoded rows and
                              ply.compressed_ply_bytes
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import torch

from . import _lib
from .ply import compressed_ply_bytes, export_comments, sh_degree_from_coeffs
from .render import RenderContext, _stream_ptr

CHUNK_ROWS = 256


class CompressedSplats(NamedTuple):
    """Device outputs of bg_compress_splats, sized for n rows; only the first `count` rows (and ceil(count/256) chunk
    rows) are written."""
    chunks: torch.Tensor            # float32 [ceil(n/256), 18]
    packed: torch.Tensor            # int32 [n, 4] (u32 words: position, rotation, scale, color)
    sh: Optional[torch.Tensor]      # uint8 [n, 3(K-1)], None when K == 1
    order: torch.Tensor             # int32 [n]: source row of each output row
    count: torch.Tensor             # int32 [1]: m, the number of kept rows


def compress_splats(ctx: RenderContext, transforms: torch.Tensor, sh: torch.Tensor, raw_opac: torch.Tensor) -> CompressedSplats:
    """Encodes transforms [n,10], sh [n,K,3], raw_opac [n] (float32 on ctx's device, the Mip floor already folded).
    Nothing is read back."""
    n, k = int(transforms.shape[0]), int(sh.shape[1])
    if transforms.shape != (n, 10) or sh.shape != (n, k, 3) or raw_opac.shape != (n,):
        raise ValueError("compress_splats needs transforms [n,10], sh [n,K,3] and raw_opac [n]")
    sh_degree_from_coeffs(k)
    dev = transforms.device
    transforms, sh, raw_opac = (x.contiguous() for x in (transforms, sh, raw_opac))
    out = CompressedSplats(
        torch.empty(((n + CHUNK_ROWS - 1) // CHUNK_ROWS, 18), dtype=torch.float32, device=dev),
        torch.empty((n, 4), dtype=torch.int32, device=dev),
        torch.empty((n, 3 * (k - 1)), dtype=torch.uint8, device=dev) if k > 1 else None,
        torch.empty(n, dtype=torch.int32, device=dev),
        torch.empty(1, dtype=torch.int32, device=dev))
    lib = _lib.load()
    need = int(lib.bg_compress_workspace_bytes(n))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    a = _lib.BgCompressArgs()
    a.n, a.k = n, k
    a.transforms, a.sh, a.raw_opac = transforms.data_ptr(), sh.data_ptr(), raw_opac.data_ptr()
    a.chunks_out, a.packed_out = out.chunks.data_ptr(), out.packed.data_ptr()
    a.sh_out = out.sh.data_ptr() if out.sh is not None else None
    a.order_out, a.count_out = out.order.data_ptr(), out.count.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), need
    _lib.check(lib.bg_compress_splats(ctx.handle, _stream_ptr(dev), C.byref(a)), "bg_compress_splats")
    return out


def splat_to_compressed_ply(ctx: RenderContext, transforms: torch.Tensor, sh: torch.Tensor, raw_opac: torch.Tensor,
                            up_axis=None, render_mip: bool = False) -> bytes:
    """The compressed counterpart of ply.splat_to_ply for device splats: the same header comments, rows with a
    non-finite value or a zero quaternion dropped, the rest in Morton order."""
    enc = compress_splats(ctx, transforms, sh, raw_opac)
    m = int(enc.count.item())                              # the one synchronise
    chunks = enc.chunks[:(m + CHUNK_ROWS - 1) // CHUNK_ROWS].cpu().numpy()
    packed = enc.packed[:m].cpu().numpy().view("u4")
    sh_bytes = enc.sh[:m].cpu().numpy() if enc.sh is not None else None
    return compressed_ply_bytes(chunks, packed, sh_bytes, m,
                                export_comments(sh_degree_from_coeffs(int(sh.shape[1])), up_axis, render_mip))
