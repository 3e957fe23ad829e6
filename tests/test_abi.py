"""CPU: libvd3d.so builds, loads, and exports every symbol include/vd3d.h declares;
ctypes structs mirror the header; no compute is called (no GPU here)."""
import ctypes as C
import os
import re

import pytest

from visiondepth3d_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        from visiondepth3d_b200 import build
        build.build()
    return _lib.load()


def _header_functions():
    src = open(os.path.join(ROOT, "include", "vd3d.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vd3d_[a-z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported(lib):
    names = _header_functions()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"{n} declared in vd3d.h but not exported"
    assert sorted(_lib.SYMBOLS) == sorted(n for n in names)


def test_struct_layouts_match_header(lib):
    # the library reports sizeof() of each ABI struct; the ctypes mirrors must agree
    for which, st in enumerate((_lib.ShiftParams, _lib.RenderParams, _lib.SizePlan, _lib.FrameInfo)):
        assert lib.vd3d_struct_size(which) == C.sizeof(st), st.__name__
    assert C.sizeof(_lib.SizePlan) == 12 * 4
    assert lib.vd3d_struct_size(99) == -1


def test_plan_sizes_matches_oracle(lib):
    from oracle import dibr as O
    from visiondepth3d_b200 import render_3d as R
    cases = [
        (1920, 1080, dict(output_width=1920, output_height=1080, output_format="Half-SBS")),
        (3840, 2160, dict(output_format="Full-SBS", preserve_original_aspect=True)),
        (3840, 2160, dict(output_height=2160, output_format="Full-SBS")),
        (1280, 720, dict(output_height=720, output_format="Red-Cyan Anaglyph")),
        (2048, 858, dict(output_height=858, output_format="Half-SBS", aspect_ratio=2.39)),
        (1440, 1080, dict(output_height=1080, output_format="Half-SBS")),  # 4:3 source, 16:9 target -> crop
        (1920, 800, dict(output_height=1080, output_format="Half-SBS")),   # wide source -> crop width
        (1920, 1080, dict(output_height=1080, output_format="VR")),        # 2 x 1440x1600 (core/render_3d.py:1129-1133)
        (1920, 1080, dict(output_format="VR", preserve_original_aspect=True)),
        (321, 180, dict(output_format="Half-SBS", preserve_original_aspect=True)),  # odd width -> 160 per eye
    ]
    # seeded sweep over sources, heights, aspects, formats and both sizing modes
    import random
    rnd = random.Random(5)
    ratios = [16 / 9, 2.39, 21 / 9, 4 / 3, 1.0, 2.35, 2.76]
    fmts = ["Half-SBS", "Full-SBS", "VR", "Red-Cyan Anaglyph", "Passive Interlaced"]
    for _ in range(300):
        sw, sh = rnd.randrange(64, 4097), rnd.randrange(64, 2305)
        cases.append((sw, sh, dict(output_width=rnd.randrange(64, 4097), output_height=rnd.randrange(64, 2305),
                                   output_format=rnd.choice(fmts), aspect_ratio=rnd.choice(ratios),
                                   preserve_original_aspect=rnd.random() < 0.5)))
    for sw, sh, kw in cases:
        orp = O.RenderParams(**kw)
        rp = R.make_render_params(orp.output_width, orp.output_height, 4.5, -1.5, -6.0, 0.2, orp.output_format,
                                  orp.aspect_ratio, 0.0, preserve_original_aspect=orp.preserve_original_aspect)
        pl = R.plan_sizes(sw, sh, rp)
        op = O.plan_sizes(sw, sh, orp)
        got = tuple(getattr(pl, f) for f, _ in _lib.SizePlan._fields_)
        exp = (op.crop_x0, op.crop_y0, op.crop_w, op.crop_h, op.target_eye_w, op.target_eye_h, op.resized_width,
               op.resized_height, op.per_eye_w, op.per_eye_h, op.out_width, op.out_height)
        assert got == exp, (sw, sh, kw)


def test_area_tables_match_cv2_restatement(lib):
    """Host half of the fractional INTER_AREA fit: the C tables equal the oracle's, which reproduce cv2.resize exactly
    (tests/test_oracle_golden.py::test_inter_area_matches_cv2)."""
    import numpy as np
    from oracle.dibr import area_tab
    for ss, ds in ((1920, 1440), (1080, 810), (1600, 1440), (640, 427), (1000, 333), (800, 799), (48, 47), (3840, 1440),
                   (321, 160), (96, 96), (96, 48)):
        cap = 16
        ofs = np.zeros(ds, np.int32)
        cnt = np.zeros(ds, np.int32)
        al = np.zeros((ds, cap), np.float32)
        T = lib.vd3d_area_table(ss, ds, ofs.ctypes.data_as(C.POINTER(C.c_int)), cnt.ctypes.data_as(C.POINTER(C.c_int)),
                                al.ctypes.data_as(C.POINTER(C.c_float)), cap)
        tab = area_tab(ss, ds)
        assert T == max(len(e) for e in tab)
        for dx, ent in enumerate(tab):
            assert cnt[dx] == len(ent) and ofs[dx] == ent[0][0], (ss, ds, dx)
            assert [e[0] for e in ent] == list(range(ofs[dx], ofs[dx] + cnt[dx]))  # consecutive sources
            assert np.array_equal(al[dx, :cnt[dx]], np.array([e[1] for e in ent], np.float32)), (ss, ds, dx)
    assert lib.vd3d_area_table(10, 20, None, None, None, 4) < 0  # enlarging is not an area shrink
    # enlarging axes: cv2's fixed-point bilinear emulation
    from oracle.dibr import _area_linear_tab
    for ss, ds in ((1280, 1920), (720, 1080), (160, 1440), (100, 133), (70, 140), (64, 65), (31, 200), (100, 80)):
        ofs = np.zeros(ds, np.int32)
        a01 = np.zeros((ds, 2), np.int32)
        assert lib.vd3d_area_linear_table(ss, ds, ofs.ctypes.data_as(C.POINTER(C.c_int)),
                                          a01.ctypes.data_as(C.POINTER(C.c_int))) == 0
        eo, ea = _area_linear_tab(ss, ds)
        assert np.array_equal(ofs, eo) and np.array_equal(a01, ea), (ss, ds)


def test_python_surface_matches_reference_signatures(golden_dir):
    """SURVEY 8(b): the drop-in keeps parameter names, order and defaults of the reference's hot-path functions
    (snapshot of the unmodified reference: tools/gen_golden.py signatures)."""
    import inspect
    import json
    import os
    from visiondepth3d_b200 import render_3d as R
    g = json.load(open(os.path.join(golden_dir, "signatures.json")))
    assert {k: float(v) for k, v in R.aspect_ratios.items()} == g.pop("aspect_ratios")
    assert len(g) == 10
    for name, ref in g.items():
        sig = inspect.signature(getattr(R, name))
        mine = [[p.name, None if p.default is inspect.Parameter.empty else repr(p.default)]
                for p in sig.parameters.values() if not p.name.startswith("_")]  # private test taps excluded
        assert mine == ref, name


def test_create_fails_loudly_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.Vd3dError, match="no CPU fallback"):
        _lib.Context(0)


def test_callers_import_lists_resolve():
    """The exact names the reference's callers import from core.render_3d / core.render_depth
    (VisionDepth3D.py:25-53, core/preview_gui.py:12-21, core/__init__.py:3-19) exist on the drop-ins."""
    from visiondepth3d_b200.render_3d import (  # noqa: F401  VisionDepth3D.py:25-38
        render_sbs_3d, format_3d_output, frame_to_tensor, depth_to_tensor, tensor_to_frame, pixel_shift_cuda,
        generate_anaglyph_3d, apply_sharpening, select_input_video, select_depth_map, select_output_video,
        process_video)
    from visiondepth3d_b200.render_depth import (  # noqa: F401  VisionDepth3D.py:41-53
        ensure_model_downloaded, update_pipeline, open_image, open_video, choose_output_directory, process_image,
        process_image_folder, process_images_in_folder, process_videos_in_folder, update_progress, cancel_requested)
    from visiondepth3d_b200.render_3d import (  # noqa: F401  core/preview_gui.py:12-21
        frame_to_tensor, depth_to_tensor, pixel_shift_cuda, apply_sharpening, tensor_to_frame, pad_to_aspect_ratio,
        format_3d_output, apply_color_grade)
    from visiondepth3d_b200.render_3d import aspect_ratios  # noqa: F401  core/__init__.py:3-10
    from visiondepth3d_b200.render_depth import process_video_folder  # noqa: F401  core/__init__.py:12-19
    import visiondepth3d_b200.render_depth as RD
    assert RD.pipe is None and RD.pipe_type is None  # module globals the callers read (core/render_depth.py:34-36)
    assert RD.ensure_model_downloaded("depth-anything/Depth-Anything-V2-Small-hf") == (None, None)  # no weights offline


def test_process_video_unwraps_gui_variables(monkeypatch, tmp_path):
    """process_video (core/render_3d.py:1594-1753): .get() unwrapping, output size per format, dispatch."""
    import cv2
    import numpy as np
    from visiondepth3d_b200 import render_3d as R

    class V:
        def __init__(self, v):
            self.v = v

        def get(self):
            return self.v

    src = str(tmp_path / "in.avi")
    wr = cv2.VideoWriter(src, cv2.VideoWriter_fourcc(*"MJPG"), 25.0, (64, 36))
    for _ in range(3):
        wr.write(np.zeros((36, 64, 3), np.uint8))
    wr.release()
    seen = {}
    monkeypatch.setattr(R, "render_sbs_3d", lambda *a, **k: seen.update(a=a, k=k))

    class W:
        def __setitem__(self, k, v):
            pass

        def update(self):
            pass

        def config(self, **k):
            pass

    args = [V(src), V("d.avi"), V("o.mp4"), V("XVID"), V(4.5), V(-1.5), V(-6.0), V(0.2), V("Full-SBS"), V("Default (16:9)"),
            R.aspect_ratios, V(10.0), V(9), W(), W(), None, None, V(False), V("H.264 / AVC (NVENC - NVIDIA GPU)"), V(23), V(True), V(True),
            V(0.02), V(False), V(0.8), V(False), V(0.01), V(True), V(True), V(False), V(0.0), V(0.0), V(True), V(0.85), V(0.5),
            V(0.05), V(0.95), V(1.2), V(1.1), V(1.0), V(1.0), 1.0, V(0.0)]
    R.process_video(*args, ipd_value=0.9, start_s=1.0, end_s=None)
    assert seen["a"][:7] == (src, "d.avi", "o.mp4", "XVID", 25.0, 128, 36)
    assert seen["a"][7:12] == (4.5, -1.5, -6.0, 0.2, "Full-SBS")
    k = seen["k"]
    assert k["selected_ffmpeg_codec"] == "h264_nvenc" and k["ipd_factor"] == 0.9 and k["start_s"] == 1.0
    assert k["original_video_width"] == 64 and k["color_contrast"] == 1.0 and k["max_pixel_shift_percent"] == 0.02
    seen.clear()
    args[8] = V("VR")       # not dispatched by the reference either
    R.process_video(*args)
    assert not seen
