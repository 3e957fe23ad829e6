"""GPU: the still-image depth path -- Pillow's bicubic resize on the device (vd3d_depth_resize_pil), mixed-source
batches in one forward (vd3d_depth_infer_images), the image drivers of render_depth against the host composition they
replace and against the images_* fixtures recorded from the reference."""
import ctypes as C
import os
import zlib

import cv2
import numpy as np
import pytest

from tests.test_image_depth_cpu import RESIZE_CASES, Var, _photo

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def weights():
    from tests.test_depth_gpu import _model
    return _model("vits")


def _engine(weights, h, w):
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine("vits", h, w)
    e.load_state_dict(weights)
    return e


@pytest.mark.parametrize("src,dst", RESIZE_CASES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in RESIZE_CASES])
def test_resize_kernel_equals_pillow(src, dst):
    from PIL import Image
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine("vits", 70, 98)  # the resize needs no weights
    a = _photo(*src, seed=src[0] * 7 + dst[1])
    assert np.array_equal(e.resize_pil(a, *dst), np.asarray(Image.fromarray(a).resize(dst, Image.BICUBIC)))
    e.close()


def _assert_cv2_cubic(u8, small):
    """u8 against cv2.resize(small, INTER_CUBIC) to its size: <= 1 LSB on < 0.2 % of the pixels
    (tests/test_oracle_golden.py::test_resize_cubic_matches_cv2)."""
    d = np.abs(u8.astype(int) - cv2.resize(small, u8.shape[::-1], interpolation=cv2.INTER_CUBIC).astype(int))
    assert d.max() <= 1 and (d > 0).mean() < 2e-3, (d.max(), (d > 0).mean())


def _bgr(a):
    return np.ascontiguousarray(a[..., ::-1])


def test_infer_images_mixed_sources_equal_single_images(weights):
    """640x480, 1024x768 and 800x600 share the processed size 518x686: one forward gives each image what it gets
    alone through DepthEngine.infer."""
    from visiondepth3d_b200.depth_engine import processed_size
    from visiondepth3d_b200.synth import synth_frame
    sizes = [(640, 480), (1024, 768), (800, 600)]
    key = processed_size(*sizes[0])
    assert all(processed_size(*s) == key for s in sizes)
    e = _engine(weights, *key)
    rgbs = [synth_frame(20 + k, w, h, "natural")[0][..., ::-1].copy() for k, (w, h) in enumerate(sizes)]
    for invert in (False, True):
        got = e.infer_images(rgbs, invert=invert, want_f32=True)
        for a, (u8, f32) in zip(rgbs, got):
            d32, d8 = e.infer(_bgr(a), invert=invert)
            assert np.array_equal(u8, d8)
            assert np.abs(f32 - d32).max() <= 1e-6 * np.abs(d32).max()
    e.close()


def test_infer_images_with_inference_size(weights):
    """With an inference size: Pillow resize, the engine's depth at that size, INTER_CUBIC back -- the host
    composition of hf_batch_safe_pipe + convert_depth_to_grayscale + the resize of the depth writer, from the engine's
    own pixels.  The resize back is the project's cv2.resize restatement (resize_cubic_u8, what the depth-video pass
    applies), which stays within 1 LSB of the installed cv2 on < 0.2 % of the pixels."""
    import torch
    from PIL import Image
    from visiondepth3d_b200 import render_depth as RD
    from visiondepth3d_b200.depth_engine import processed_size
    from visiondepth3d_b200.synth import synth_frame
    inf = (384, 384)
    e = _engine(weights, *processed_size(*inf))
    sizes = [(640, 480), (1024, 768), (800, 600), (333, 517), (384, 384)]
    rgbs = [synth_frame(30 + k, w, h, "natural")[0][..., ::-1].copy() for k, (w, h) in enumerate(sizes)]
    got = e.infer_images(rgbs, [inf] * len(rgbs), invert=True, want_f32=True)
    for a, (u8, f32) in zip(rgbs, got):
        small = np.asarray(Image.fromarray(a).resize(inf, Image.BICUBIC))
        d32, d8 = e.infer(_bgr(small), invert=True)
        want = d8 if small.shape == a.shape else RD.resize_cubic_u8(d8, a.shape[1], a.shape[0])
        assert np.array_equal(u8, want)
        _assert_cv2_cubic(u8, d8)
        assert np.abs(f32 - d32).max() <= 1e-6 * np.abs(d32).max()
    # device memory: the same bits
    dev = e.infer_images([torch.from_numpy(a).cuda() for a in rgbs], [inf] * len(rgbs), invert=True, want_f32=True)
    for (u8, f32), (du8, df32) in zip(got, dev):
        assert np.array_equal(du8.cpu().numpy(), u8) and np.array_equal(df32.cpu().numpy(), f32)
    e.close()


def test_infer_images_refuses_other_processed_sizes(weights):
    from visiondepth3d_b200 import _lib
    e = _engine(weights, 518, 686)
    a = np.zeros((854, 480, 3), np.uint8)
    with pytest.raises(ValueError, match="processed size"):
        e.infer_images([np.zeros((480, 640, 3), np.uint8), a])
    sizes = np.array([[854, 480, 854, 480]], np.int32)
    out = np.empty((854, 480), np.uint8)
    rc = e.lib.vd3d_depth_infer_images(e.h, 1, (C.c_void_p * 1)(a.ctypes.data), sizes.ctypes.data_as(
        C.POINTER(C.c_int32)), (C.c_void_p * 1)(out.ctypes.data), None, 0, _lib.MEM_HOST)
    assert rc == -2 and b"processed size" in e.lib.vd3d_depth_last_error(e.h)
    e.close()


@pytest.fixture
def loaded(weights, monkeypatch):
    from visiondepth3d_b200 import render_depth as RD
    RD.load_depth_model("vits", weights, 640, 480)
    monkeypatch.setattr(RD, "USE_TILED_DEPTH", False)
    RD.cancel_requested.clear()
    return RD


def _host_composition(RD, path, inference_size, invert):
    """What the folder driver replaces: hf_batch_safe_pipe -> convert_depth_to_grayscale -> invert -> INTER_CUBIC back
    to the image size (resize_cubic_u8, as the depth-video pass does it; checked against cv2 itself)."""
    from PIL import Image
    img = Image.open(path).convert("RGB")
    d8 = RD.convert_depth_to_grayscale(RD.hf_batch_safe_pipe([img], inference_size)[0]["predicted_depth"])
    if invert:
        d8 = 255 - d8
    if d8.shape[::-1] == img.size:
        return d8.copy()
    out = RD.resize_cubic_u8(d8, *img.size)
    _assert_cv2_cubic(out, d8)
    return out


@pytest.mark.parametrize("res,invert", [("Original", False), ("384x384", True), ("910x518 (Depth Anything)", False)])
def test_folder_driver_equals_host_composition(loaded, tmp_path, res, invert):
    from PIL import Image
    from visiondepth3d_b200.synth import image_folder
    RD = loaded
    src = image_folder(str(tmp_path / "in"))
    RD.process_images_in_folder(src, Var("8"), Var(str(tmp_path / "o")), Var(res), None, None, None, Var(invert))
    inf = RD.parse_inference_resolution(res)
    names = [f for f in os.listdir(src) if f.lower().endswith((".jpeg", ".jpg", ".png"))]
    assert len(names) == 4
    for f in names:
        want = tmp_path / ("want_" + f + ".png")
        Image.fromarray(_host_composition(RD, os.path.join(src, f), inf, invert)).save(want)
        got = tmp_path / "o" / (os.path.splitext(f)[0] + "_depth.png")
        assert got.read_bytes() == want.read_bytes(), f
        # process_image writes the same file
        RD.process_image(os.path.join(src, f), Var("default"), Var(invert), Var(str(tmp_path / "s")), Var(res), None,
                         None, None, None)
        assert (tmp_path / "s" / got.name).read_bytes() == got.read_bytes(), f


def test_tiled_branch_equals_tile_path(loaded, tmp_path, monkeypatch):
    from PIL import Image
    from visiondepth3d_b200.synth import image_folder
    RD = loaded
    monkeypatch.setattr(RD, "USE_TILED_DEPTH", True)
    src = image_folder(str(tmp_path / "in"))
    for res in ("Original", "256x256"):  # (infer_depth_tile refuses sizes that shrink one axis and enlarge the other)
        out = tmp_path / res
        RD.process_images_in_folder(src, Var("8"), Var(str(out)), Var(res), None, None, None, Var(True))
        inf = RD.parse_inference_resolution(res)
        for f in ("b_street.JPG", "d_odd.jpeg"):
            img = Image.open(os.path.join(src, f)).convert("RGB")
            dep = RD.infer_depth_tile(RD.pipe, np.array(img), inf)
            want = RD._normalize_to_u8(dep, img.size, invert=True)
            got = np.asarray(Image.open(out / (os.path.splitext(f)[0] + "_depth.png")))
            assert np.array_equal(got, want), (res, f)


@pytest.mark.parametrize("tag", ["original", "384x384", "invert"])
def test_reference_fixtures(loaded, tmp_path, tag):
    """File names, shapes and mode equal the reference's; the u8 values agree within 2e-2 of the range (+1 LSB of
    truncation), the bound the end-to-end HF test puts on the depth (random-init weights, f16 tensor cores against
    the reference's fp32 CPU forward)."""
    from PIL import Image
    from visiondepth3d_b200.synth import IMAGE_FOLDER, image_folder
    RD = loaded
    g = np.load(os.path.join(GOLDEN, f"images_{tag}.npz"))
    src = image_folder(str(tmp_path / "in"))
    crc = [zlib.crc32(np.asarray(Image.open(os.path.join(src, n)).convert("RGB")).tobytes()) for n, *_ in IMAGE_FOLDER]
    assert np.array_equal(np.array(crc, np.uint32), g["input_crc"])  # same decoded photos as at recording
    RD.process_images_in_folder(src, Var("4"), Var(str(tmp_path / "o")), Var(str(g["resolution"])), None, None, None,
                                Var(bool(g["invert"])))
    names = sorted(os.listdir(tmp_path / "o"))
    assert names == list(g["folder_names"]) == list(g["single_names"])
    worst = 0
    for n in names:
        im = Image.open(tmp_path / "o" / n)
        assert im.mode == str(g[f"folder_mode_{n}"]) == "L"
        a = np.asarray(im)
        assert list(a.shape) == list(g[f"shape_{n}"])
        worst = max(worst, int(np.abs(a[::4, ::4].astype(int) - g[f"u8_{n}"].astype(int)).max()))
    print(f"images_{tag}: max |u8 - reference| = {worst} LSB")
    assert worst <= 6
