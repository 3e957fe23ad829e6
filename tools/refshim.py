"""Import shim for the UNMODIFIED reference (a VisionDepth3D checkout named by $VD3D_REFERENCE).

Test infrastructure only: used in the build container by tools/gen_golden.py to
produce tests/golden/*.npz and to pin oracle/ against the real reference.
Nothing here (and nothing in the reference checkout) is needed at run time on
the GPU.  Recipe follows SURVEY.md section 8(c): stub GUI / ORT modules with a
real __spec__, register a bare `core` package so core/__init__.py never runs.
"""
import importlib
import importlib.machinery
import os
import sys
import types

REF_ROOT = os.environ.get("VD3D_REFERENCE", "")


class _Anything(types.ModuleType):
    """Module whose attributes are manufactured on demand (empty classes)."""

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        obj = type(name, (), {"__init__": lambda self, *a, **k: None})
        setattr(self, name, obj)
        return obj


def _stub(name, is_pkg=False):
    if name in sys.modules:
        return sys.modules[name]
    m = _Anything(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, None, is_package=is_pkg)
    if is_pkg:
        m.__path__ = []
    sys.modules[name] = m
    parent, _, child = name.rpartition(".")
    if parent and parent in sys.modules:
        setattr(sys.modules[parent], child, m)
    return m


def load_reference(modules=("render_3d",)):
    """Return {name: module} for core.<name>, reference files untouched."""
    if not REF_ROOT or not os.path.isdir(os.path.join(REF_ROOT, "core")):
        raise SystemExit("set VD3D_REFERENCE to a VisionDepth3D checkout (the directory holding core/render_3d.py); "
                         f"got {REF_ROOT!r}")
    import PIL  # real

    for n in ("tkinter", "tkinter.filedialog", "tkinter.messagebox",
              "tkinter.simpledialog", "tkinter.ttk", "onnxruntime"):
        _stub(n, is_pkg=(n == "tkinter"))
    it = _stub("PIL.ImageTk")
    PIL.ImageTk = it
    if "render_depth" in modules:
        for n in ("matplotlib", "matplotlib.cm", "matplotlib.pyplot"):
            _stub(n, is_pkg=(n == "matplotlib"))
        try:
            import diffusers  # noqa: F401
        except Exception:
            for n in ("diffusers", "diffusers.models", "diffusers.utils",
                      "diffusers.models.unets", "diffusers.models.unets.unet_spatio_temporal_condition",
                      "diffusers.pipelines", "diffusers.pipelines.stable_video_diffusion",
                      "diffusers.pipelines.stable_video_diffusion.pipeline_stable_video_diffusion",
                      "diffusers.utils.torch_utils", "diffusers.schedulers", "diffusers.image_processor"):
                _stub(n, is_pkg=True)
    if "core" not in sys.modules:
        core = types.ModuleType("core")
        core.__path__ = [REF_ROOT + "/core"]
        core.__spec__ = importlib.machinery.ModuleSpec(
            "core", None, is_package=True)
        core.__spec__.submodule_search_locations = core.__path__
        sys.modules["core"] = core
    out = {}
    for m in modules:
        out[m] = importlib.import_module("core." + m)
    return out


def reset_singletons(r3d):
    """Reset module-level temporal state (core/render_3d.py:284-285,500,511)."""
    r3d.depth_ema_norm._lo = None
    r3d.depth_ema_norm._hi = None
    r3d.conv_ema.val = None
    r3d.floating_window_tracker.prev_offset = 0.0
    r3d.floating_window_tracker.frame_counter = 0
    r3d.bar_easer.prev_bar_width = 0
