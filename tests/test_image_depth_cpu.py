"""CPU: the still-image depth path without a GPU -- the Pillow bicubic restatement (oracle/pil_resize.py) and the
library's host-built tables against Pillow, parse_inference_resolution against the reference's resolution choices,
and the image drivers of render_depth with a stand-in for the engine call (file discovery, output names, the output
directory, cancellation, progress, per-file errors, grouping by processed size)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import pil_resize as P

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")

# (source (W, H), output (W, H)): shrink, enlarge, one axis unchanged either way, shrink one axis while enlarging the
# other, 1-pixel outputs, odd sizes, a 12 MP photo to a square inference size
RESIZE_CASES = [((640, 480), (320, 240)), ((100, 80), (250, 170)), ((333, 517), (333, 300)), ((333, 517), (500, 517)),
                ((400, 300), (200, 500)), ((97, 53), (1, 1)), ((97, 53), (1, 40)), ((53, 97), (40, 1)),
                ((13, 7), (29, 3)), ((517, 333), (384, 384)), ((1, 1), (5, 3)), ((4032, 3024), (896, 896))]


def _photo(w, h, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    a[: h // 3] = 0            # flat black and white bands: the clip at both ends of 0..255
    a[h // 3: h // 2] = 255
    return a


@pytest.mark.parametrize("src,dst", RESIZE_CASES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in RESIZE_CASES])
def test_pil_restatement_equals_pillow(src, dst):
    from PIL import Image
    a = _photo(*src, seed=src[0] * 7 + dst[1])
    assert np.array_equal(P.resize(a, dst), np.asarray(Image.fromarray(a).resize(dst, Image.BICUBIC)))
    g = a[..., 1].copy()  # mode "L"
    assert np.array_equal(P.resize(g, dst), np.asarray(Image.fromarray(g).resize(dst, Image.BICUBIC)))


@pytest.fixture(scope="module")
def lib():
    from visiondepth3d_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from visiondepth3d_b200 import build
        build.build()
    from visiondepth3d_b200.depth_engine import _bind
    lib = _lib.load()
    _bind(lib)
    return lib


@pytest.mark.parametrize("n_in,n_out", [(640, 320), (100, 250), (97, 1), (13, 29), (517, 384), (4032, 896), (3024, 896),
                                        (1, 5), (1080, 686)])
def test_host_tables_equal_restatement(lib, n_in, n_out):
    xmin, cnt, kk = P.coeffs(n_in, n_out)
    ksize = lib.vd3d_pil_bicubic_table(n_in, n_out, None, None, 0)
    assert ksize == kk.shape[1]
    bounds = np.zeros((n_out, 2), np.int32)
    got = np.zeros((n_out, ksize), np.int32)
    assert lib.vd3d_pil_bicubic_table(n_in, n_out, bounds.ctypes.data, got.ctypes.data, ksize) == ksize
    assert np.array_equal(bounds[:, 0], xmin) and np.array_equal(bounds[:, 1], cnt)
    assert np.array_equal(got, kk)
    assert lib.vd3d_pil_bicubic_table(n_in, n_out, bounds.ctypes.data, got.ctypes.data, ksize - 1) < 0


def test_parse_inference_resolution_matches_reference_choices():
    from visiondepth3d_b200.render_depth import parse_inference_resolution
    table = json.load(open(os.path.join(GOLDEN, "images_resolutions.json")))
    assert len(table) >= 30 and table["Original"] is None
    for key, want in table.items():
        assert parse_inference_resolution(key) == (tuple(want) if want else None), key
        assert parse_inference_resolution(f"  {key} ") == (tuple(want) if want else None), key
    assert parse_inference_resolution("Automatic") == (384, 384)
    assert parse_inference_resolution("bogus", fallback=None) is None


@pytest.mark.skipif(not os.environ.get("VD3D_REFERENCE"), reason="needs a reference checkout ($VD3D_REFERENCE)")
def test_parse_inference_resolution_against_live_reference():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(GOLDEN), "..", "tools"))
    import refshim
    for n in ("diffusers.configuration_utils", "core.unet", "core.depthcrafter_adapter"):
        refshim._stub(n)
    rd = refshim.load_reference(("render_depth",))["render_depth"]
    from visiondepth3d_b200.render_depth import parse_inference_resolution
    for key, want in rd.INFERENCE_RESOLUTIONS.items():
        assert parse_inference_resolution(key) == want, key
    assert parse_inference_resolution("bogus") == rd.parse_inference_resolution("bogus")


class Var:
    def __init__(self, v):
        self.v = v

    def get(self):
        return self.v


class Widget:
    def __init__(self):
        self.texts = []
        self.kw = {}

    def config(self, **kw):
        self.kw.update(kw)
        if "text" in kw:
            self.texts.append(kw["text"])


class FakeEngine:
    """Stand-in for the depth engine: records each infer_images call; the depth of an image is a constant plane."""

    def __init__(self, calls, key, hook=None):
        self.calls, self.key, self.hook = calls, key, hook

    def infer_images(self, rgbs, input_sizes, invert=False):
        self.calls.append((self.key, [(a.shape[1], a.shape[0]) for a in rgbs], list(input_sizes), invert))
        if self.hook:
            self.hook(len(self.calls))
        out = []
        for a in rgbs:
            v = int(a.shape[1] % 200)
            out.append((np.full(a.shape[:2], 255 - v if invert else v, np.uint8), None))
        return out


@pytest.fixture
def stub_engine(monkeypatch):
    from visiondepth3d_b200 import render_depth as RD
    from visiondepth3d_b200.depth_engine import processed_size
    calls = []
    state = {"hook": None}
    monkeypatch.setattr(RD, "_engine_for", lambda w, h: FakeEngine(calls, processed_size(w, h), state["hook"]))
    monkeypatch.setattr(RD, "USE_TILED_DEPTH", False)
    progress = []
    monkeypatch.setattr(RD, "update_progress", lambda *a: progress.append(a[:2]))
    RD.cancel_requested.clear()
    yield RD, calls, progress, state
    RD.cancel_requested.clear()


def _folder(tmp_path):
    from visiondepth3d_b200.synth import image_folder
    return image_folder(str(tmp_path / "in"))


def test_folder_driver_discovery_names_and_grouping(stub_engine, tmp_path):
    from PIL import Image
    from visiondepth3d_b200.depth_engine import processed_size
    from visiondepth3d_b200.synth import IMAGE_FOLDER
    RD, calls, progress, _ = stub_engine
    src = _folder(tmp_path)
    out = tmp_path / "out" / "nested"  # created by the driver
    status = Widget()
    RD.process_images_in_folder(src, Var("8"), Var(str(out)), Var("Original"), status, Widget(), None, Var(False))
    order = [f for f in os.listdir(src) if f.lower().endswith((".jpeg", ".jpg", ".png"))]
    assert sorted(os.listdir(out)) == sorted(os.path.splitext(f)[0] + "_depth.png" for f in order)
    sizes = {name: (w, h) for name, w, h, _ in IMAGE_FOLDER}
    for f in order:
        im = Image.open(out / (os.path.splitext(f)[0] + "_depth.png"))
        assert im.mode == "L" and im.size == sizes[f]
        assert (np.asarray(im) == sizes[f][0] % 200).all()
    # one engine call per processed size: the two landscape shots (640x480, 1024x768) share one forward
    groups = {}
    for f in order:
        groups.setdefault(processed_size(*sizes[f]), []).append(sizes[f])
    assert sorted((k, s) for k, s, _, _ in calls) == sorted(groups.items())
    assert sum(len(s) == 2 for _, s, _, _ in calls) == 1
    assert progress == [(k, 4) for k in range(1, 5)]
    assert status.texts[0] == "📂 Processing 4 images..." and status.texts[-1] == "✅ All images processed successfully!"


def test_folder_driver_inference_size_batches_and_invert(stub_engine, tmp_path):
    RD, calls, progress, _ = stub_engine
    src = _folder(tmp_path)
    RD.process_images_in_folder(src, Var("3"), Var(str(tmp_path / "o")), Var("384x384"), None, None, None, Var(True))
    # chunks of the batch size (3 + 1), each one forward: every image maps to the 384x384 input's processed size
    assert [len(s) for _, s, _, _ in calls] == [3, 1]
    assert all(ins == [(384, 384)] * len(s) and inv for _, s, ins, inv in calls)
    assert len(os.listdir(tmp_path / "o")) == 4


def test_folder_driver_output_directory_and_empty_folder(stub_engine, tmp_path, capsys):
    RD, calls, _, _ = stub_engine
    src = _folder(tmp_path)
    status = Widget()
    RD.process_images_in_folder(src, Var("4"), Var("  "), Var("Original"), status, None, None, Var(False))
    assert status.texts == ["❌ Output directory not selected."] and not calls
    assert "Please select an output directory" in capsys.readouterr().out
    blocker = tmp_path / "file"
    blocker.write_text("x")
    RD.process_images_in_folder(src, Var("4"), Var(str(blocker / "sub")), Var("Original"), status, None, None, Var(False))
    assert status.texts[-1] == "❌ Failed to create output directory." and not calls
    empty = tmp_path / "empty"
    empty.mkdir()
    RD.process_images_in_folder(str(empty), Var("4"), Var(str(tmp_path / "o")), Var("Original"), status, None, None,
                                Var(False))
    assert status.texts[-1] == "⚠️ No image files found."
    RD.process_images_in_folder(src, Var("zero"), Var(str(tmp_path / "o")), Var("Original"), status, None, None,
                                Var(False))
    assert any(t.startswith("⚠️ Invalid batch size. Using dynamic batch size: ") for t in status.texts)


def test_folder_driver_cancellation(stub_engine, tmp_path):
    RD, calls, _, state = stub_engine
    src = _folder(tmp_path)
    status = Widget()
    RD.cancel_requested.set()
    RD.process_images_in_folder(src, Var("2"), Var(str(tmp_path / "a")), Var("Original"), status, None, None, Var(False))
    assert status.texts[-1] == "❌ Cancelled by user." and not calls and not os.listdir(tmp_path / "a")
    RD.cancel_requested.clear()
    state["hook"] = lambda n: RD.cancel_requested.set()  # cancel while the first batch is in flight
    RD.process_images_in_folder(src, Var("2"), Var(str(tmp_path / "b")), Var("Original"), status, None, None, Var(False))
    assert status.texts[-1] == "❌ Cancelled during batch." and not os.listdir(tmp_path / "b")


def test_folder_driver_reports_a_bad_file_and_continues(stub_engine, tmp_path, monkeypatch, capsys):
    RD, calls, progress, _ = stub_engine
    src = _folder(tmp_path)
    real = RD.depth_images
    monkeypatch.setattr(RD, "depth_images", lambda imgs, inf, inv: [None] + real(imgs, inf, inv)[1:])
    RD.process_images_in_folder(src, Var("8"), Var(str(tmp_path / "o")), Var("Original"), Widget(), Widget(), None,
                                Var(False))
    first = [f for f in os.listdir(src) if f.lower().endswith((".jpeg", ".jpg", ".png"))][0]
    assert f"❌ Error processing {os.path.join(src, first)}:" in capsys.readouterr().out
    assert len(os.listdir(tmp_path / "o")) == 3 and len(progress) == 3


def test_process_image_writes_the_folder_file(stub_engine, tmp_path, capsys):
    RD, calls, _, _ = stub_engine
    src = _folder(tmp_path)
    RD.process_images_in_folder(src, Var("8"), Var(str(tmp_path / "f")), Var("Original"), None, None, None, Var(True))
    status, bar = Widget(), Widget()
    for name in ("b_street.JPG", "d_odd.jpeg"):
        RD.process_image(os.path.join(src, name), Var("Default"), Var(True), Var(str(tmp_path / "s")), Var("Original"),
                         None, None, status, bar)
        out = os.path.splitext(name)[0] + "_depth.png"
        assert (tmp_path / "s" / out).read_bytes() == (tmp_path / "f" / out).read_bytes()
        assert status.texts[-1] == f"✅ Image saved: {tmp_path / 's' / out}" and bar.kw["value"] == 100
    RD.process_image(os.path.join(src, "d_odd.jpeg"), Var("Viridis"), Var(True), Var(str(tmp_path / "c")),
                     Var("Original"), None, None, None, None)
    assert "⚠️ Unknown colormap 'viridis', defaulting to grayscale." in capsys.readouterr().out
    assert (tmp_path / "c" / "d_odd_depth.png").read_bytes() == (tmp_path / "f" / "d_odd_depth.png").read_bytes()


def test_dialog_drivers(stub_engine, tmp_path, monkeypatch):
    import sys
    RD, calls, _, _ = stub_engine
    src = _folder(tmp_path)
    picks = iter([os.path.join(src, "a_room.png"), src, "", ""])
    monkeypatch.setattr(RD, "_dialog", lambda kind, **kw: next(picks))
    RD.open_image(None, None, Var("Default"), Var(False), Var(str(tmp_path / "o")), Var("Original"), None, None).join()
    assert os.listdir(tmp_path / "o") == ["a_room_depth.png"]
    RD.process_image_folder(Var("8"), Var(str(tmp_path / "o")), Var("Original"), None, None, Var(False), None).join()
    assert len(os.listdir(tmp_path / "o")) == 4
    status = Widget()
    assert RD.process_image_folder(Var("8"), Var(""), Var("Original"), status, None, Var(False), None) is None
    assert status.texts == ["⚠️ No folder selected."]
    assert RD.open_image(status, None, Var("Default"), Var(False), Var(""), Var("Original"), None, None) is None
    # without tkinter the dialogs raise the GUI helper's error
    monkeypatch.undo()
    monkeypatch.setitem(sys.modules, "tkinter", None)
    monkeypatch.setitem(sys.modules, "tkinter.filedialog", None)
    with pytest.raises(RuntimeError, match="tkinter"):
        RD.open_image(None, None, Var("Default"), Var(False), Var(""), Var("Original"), None, None)
    with pytest.raises(RuntimeError, match="tkinter"):
        RD.process_image_folder(Var("8"), Var(""), Var("Original"), None, None, Var(False), None)


def test_depth_images_groups_by_processed_size(stub_engine):
    RD, calls, _, _ = stub_engine
    imgs = [np.zeros((480, 640, 3), np.uint8), np.zeros((854, 480, 3), np.uint8), np.zeros((768, 1024, 3), np.uint8)]
    imgs += [np.zeros((600, 800, 3), np.uint8)] * 7
    out = RD.depth_images(imgs)
    assert [o.shape for o in out] == [a.shape[:2] for a in imgs]
    # nine 4:3 images: chunks of 8 + 1; the portrait alone
    assert sorted(len(s) for _, s, _, _ in calls) == [1, 1, 8]
