"""Depth supervision in the multi-view step on the host (DESIGN.md section 4.7): the header declares the two entry points,
their C prototypes agree with the ctypes signatures, and SplatTrainer rejects what it must before anything runs on a
device.  No GPU needed."""
import ctypes
import os
import re
import subprocess
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the C prototypes the ctypes signatures stand for
PROTOTYPES = {
    "bg_train_step_views_depth_workspace_bytes": ("uint64_t", ["uint32_t"] * 6),
    "bg_train_step_views_depth": ("int32_t", ["BgContext *", "BgDpComm *", "void *", "BgTrainViewsArgs *",
                                              "const BgDepthSupervision *"]),
}


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "brush_b200.h")).read(), flags=re.S)


def test_header_declares_the_views_depth_entry_points():
    hdr = _header()
    for name in PROTOTYPES:
        assert re.search(r"\b%s\s*\(" % name, hdr), name


def _ctype_of(c_type: str):
    from brush_b200 import _lib
    scalars = {"uint32_t": ctypes.c_uint32, "uint64_t": ctypes.c_uint64, "int32_t": ctypes.c_int32}
    if c_type in scalars:
        return scalars[c_type]
    struct = c_type.replace("const", "").replace("*", "").strip()
    if struct in ("BgContext", "BgDpComm", "void"):
        return ctypes.c_void_p                                   # opaque handles and the stream
    return ctypes.POINTER(getattr(_lib, struct))


def test_ctypes_signatures_match_a_c_program_built_against_the_header(tmp_path):
    """The prototypes compile as exact function-pointer types against the header (-Werror: any parameter or return type
    that differs fails), and the ctypes signatures are their mirror; the BgDepthSupervision array stride agrees."""
    from brush_b200 import _lib
    prog = ["#include <stdio.h>", '#include "brush_b200.h"']
    for name, (res, args) in PROTOTYPES.items():
        prog.append(f"typedef {res} (*{name}_fn)({', '.join(args)});")
    prog.append("int main(void) {")
    for name in PROTOTYPES:
        prog.append(f"    {name}_fn p_{name} = {name}; (void)p_{name};")
    prog.append('    printf("%zu %zu\\n", sizeof(BgDepthSupervision), sizeof(BgTrainViewsArgs));')
    prog.append("    return 0;\n}")
    src = tmp_path / "views_depth_proto.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "views_depth_proto"
    r = subprocess.run(["gcc", "-Werror", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                        "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sizes = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert int(sizes[0]) == ctypes.sizeof(_lib.BgDepthSupervision)
    assert int(sizes[1]) == ctypes.sizeof(_lib.BgTrainViewsArgs)
    for name, (res, args) in PROTOTYPES.items():
        want_res, want_args = _lib.SIGNATURES[name]
        assert want_res == _ctype_of(res), name
        assert list(want_args) == [_ctype_of(a) for a in args], name


def _host_trainer(weight):
    """A trainer whose checks run on the host: CPU tensors and a context that only names the device."""
    import brush_b200.train as T
    from brush_b200.camera import Camera
    cfg = T.TrainConfig(total_train_iters=100, depth_loss_weight=weight)
    t = T.SplatTrainer(cfg, types.SimpleNamespace(device="cpu"), T.BoundingBox(torch.zeros(3).numpy(), torch.ones(3).numpy()))
    s = T.Splats(torch.zeros(4, 10), torch.zeros(4, 1, 3), torch.zeros(4))
    img = torch.zeros((6, 8), dtype=torch.int32)
    return T, t, s, img, Camera(position=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0))


def test_step_views_refusal_names_step_views_depth():
    T, t, s, img, cam = _host_trainer(0.5)
    b = T.SceneBatch(img_packed=img, camera=cam, depth=torch.ones(6, 8), depth_count=48)
    with pytest.raises(ValueError, match="step_views_depth"):
        t.step_views([b], s, distributed=False)
    assert t.step_count == 0


def test_step_views_depth_rejects_a_misshaped_depth_map_before_the_step():
    T, t, s, img, cam = _host_trainer(0.5)
    good = T.SceneBatch(img_packed=img, camera=cam, depth=torch.ones(6, 8), depth_count=48)
    for shape, count in (((6, 9), 54), ((8, 6), 48), ((6, 8, 1), 48), ((6, 9), 0)):
        bad = T.SceneBatch(img_packed=img, camera=cam, depth=torch.ones(shape), depth_count=count)
        with pytest.raises(ValueError, match="depth"):
            t.step_views_depth([good, bad], s, distributed=False)
    assert t.step_count == 0
    with pytest.raises(ValueError):
        t.step_views_depth([], s, distributed=False)
