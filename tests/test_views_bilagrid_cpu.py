"""Bilateral grids in the multi-view step on the host (DESIGN.md section 4.11): the header declares the three entry points,
their C prototypes and the BgBilagridViews layout agree with the ctypes mirror, and SplatTrainer.step_views_bilagrid
rejects what it must before anything runs on a device.  No GPU needed."""
import ctypes
import os
import re
import subprocess
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROTOTYPES = {
    "bg_train_step_views_bilagrid_workspace_bytes": ("uint64_t", ["uint32_t"] * 6),
    "bg_train_step_views_bilagrid": ("int32_t", ["BgContext *", "BgDpComm *", "void *", "BgTrainViewsArgs *",
                                                 "const BgDepthSupervision *", "const BgBilagridViews *"]),
    "bg_bilagrid_update_views": ("int32_t", ["BgContext *", "void *", "const BgBilagridViews *", "uint32_t", "const uint32_t *",
                                             "float *"]),
}
FIELDS = ("grids", "m", "v", "steps", "num_views", "view_index", "lr", "tv_weight", "tv_loss_out")


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "brush_b200.h")).read(), flags=re.S)


def test_header_declares_the_views_bilagrid_entry_points():
    hdr = _header()
    for name in PROTOTYPES:
        assert re.search(r"\b%s\s*\(" % name, hdr), name


def _ctype_of(c_type: str):
    from brush_b200 import _lib
    scalars = {"uint32_t": ctypes.c_uint32, "uint64_t": ctypes.c_uint64, "int32_t": ctypes.c_int32}
    if c_type in scalars:
        return scalars[c_type]
    struct = c_type.replace("const", "").replace("*", "").strip()
    if struct in ("BgContext", "BgDpComm", "void", "uint32_t", "float"):
        return ctypes.c_void_p                                   # opaque handles, the stream and device arrays
    return ctypes.POINTER(getattr(_lib, struct))


def test_prototypes_and_layout_match_a_c_program_built_against_the_header(tmp_path):
    from brush_b200 import _lib
    prog = ["#include <stdio.h>", "#include <stddef.h>", '#include "brush_b200.h"']
    for name, (res, args) in PROTOTYPES.items():
        prog.append(f"typedef {res} (*{name}_fn)({', '.join(args)});")
    prog.append("int main(void) {")
    for name in PROTOTYPES:
        prog.append(f"    {name}_fn p_{name} = {name}; (void)p_{name};")
    prog.append('    printf("%zu", sizeof(BgBilagridViews));')
    for f in FIELDS:
        prog.append(f'    printf(" %zu", offsetof(BgBilagridViews, {f}));')
    prog.append('    printf("\\n");\n    return 0;\n}')
    src = tmp_path / "views_bilagrid_proto.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "views_bilagrid_proto"
    r = subprocess.run(["gcc", "-Werror", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                        "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = _lib.BgBilagridViews
    assert got == [ctypes.sizeof(S)] + [getattr(S, f).offset for f in FIELDS]
    for name, (res, args) in PROTOTYPES.items():
        want_res, want_args = _lib.SIGNATURES[name]
        assert want_res == _ctype_of(res), name
        assert list(want_args) == [_ctype_of(a) for a in args], name


def _host_trainer(grids_device="cpu"):
    """A trainer whose checks run on the host: CPU tensors and a context that only names the device."""
    import brush_b200.bilagrid as B
    import brush_b200.train as T
    from brush_b200.camera import Camera
    cfg = T.TrainConfig(total_train_iters=100, bilateral_grid=True)
    grids = B.BilateralGrids(3, grids_device)
    t = T.SplatTrainer(cfg, types.SimpleNamespace(device=torch.device("cpu")),
                       T.BoundingBox(torch.zeros(3).numpy(), torch.ones(3).numpy()), bilateral_grids=grids)
    s = T.Splats(torch.zeros(4, 10), torch.zeros(4, 1, 3), torch.zeros(4))
    img = torch.zeros((6, 8), dtype=torch.int32)
    return T, t, s, img, Camera(position=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0))


def test_argument_errors_are_raised_before_the_step():
    T, t, s, img, cam = _host_trainer()
    ok = T.SceneBatch(img_packed=img, camera=cam, view_index=2)
    for bad_index in (3, 7, -1):
        with pytest.raises(ValueError, match="view"):
            t.step_views_bilagrid([ok, T.SceneBatch(img_packed=img, camera=cam, view_index=bad_index)], s, distributed=False)
    with pytest.raises(ValueError, match="view_index"):
        t.step_views_bilagrid([T.SceneBatch(img_packed=img, camera=cam)], s, distributed=False)   # no view_index
    with pytest.raises(ValueError):
        t.step_views_bilagrid([], s, distributed=False)
    assert t.step_count == 0 and t.bilateral_grids.steps == [0, 0, 0]


def test_grids_on_another_device_are_refused():
    T, t, s, img, cam = _host_trainer()
    t.ctx = types.SimpleNamespace(device=torch.device("cuda", 0))
    with pytest.raises(ValueError, match="device"):
        t.step_views_bilagrid([T.SceneBatch(img_packed=img, camera=cam, view_index=0)], s, distributed=False)
    assert t.step_count == 0


def test_step_views_refusal_names_step_views_bilagrid():
    T, t, s, img, cam = _host_trainer()
    b = T.SceneBatch(img_packed=img, camera=cam, view_index=0)
    for step in (t.step_views, t.step_views_depth):
        with pytest.raises(ValueError, match="bilateral grids.*step_views_bilagrid"):
            step([b], s, distributed=False)
    assert t.step_count == 0


def test_step_views_bilagrid_needs_grids():
    import brush_b200.train as T
    from brush_b200.camera import Camera
    t = T.SplatTrainer(T.TrainConfig(total_train_iters=100), types.SimpleNamespace(device=torch.device("cpu")),
                       T.BoundingBox(torch.zeros(3).numpy(), torch.ones(3).numpy()))
    s = T.Splats(torch.zeros(4, 10), torch.zeros(4, 1, 3), torch.zeros(4))
    b = T.SceneBatch(img_packed=torch.zeros((6, 8), dtype=torch.int32), camera=Camera(position=(0.0, 0.0, 0.0),
                     rotation=(0.0, 0.0, 0.0, 1.0)), view_index=0)
    with pytest.raises(ValueError, match="bilateral_grid"):
        t.step_views_bilagrid([b], s, distributed=False)


def test_host_and_device_counts_follow_each_other_on_the_host():
    """The count bookkeeping without a device: single-view steps advance the host list, a multi-view step hands out the
    device counts (brought up to date once) and the list is read back from them once."""
    import brush_b200.bilagrid as B
    g = B.BilateralGrids(3, "cpu")
    g.step_args(1, 1e-3, 10.0)
    g.step_args(1, 1e-3, 10.0)
    assert g.steps == [0, 2, 0]
    dev = g.advance_on_device()
    assert dev.tolist() == [0, 2, 0]                     # written from the host list
    dev[0] += 1                                          # what a multi-view step of view 0 does on the device
    assert g.steps == [1, 2, 0]                          # read back
    a = g.step_args(0, 1e-3, 10.0)
    assert a.step == 2 and g.steps == [2, 2, 0]
    assert g.device_steps.tolist() == [2, 2, 0]
