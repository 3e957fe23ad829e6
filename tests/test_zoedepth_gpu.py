"""GPU: ZoeDepth on the depth engine -- each new kernel against float64 (or transformers' processor) through the
vd3d_zoe_kernel hook, the forward against tests/zoedepth_oracle.py (fp32) for the two-configuration head on both routes
and the single-configuration head, per-image routing inside a batch, the family's argument checks and the post-process
crop of the drivers."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import hybrid_zoe_kernel_refs as HZ
from tests import zoedepth_oracle as ZO

pytestmark = pytest.mark.gpu

# Gates.  The forward: 1.5e-3 of the depth range, dpt-beit-large-512's gate (the f16 trunk sets the floor; the head's
# f16 weights alone move the oracle by far less, tests/test_zoedepth_cpu.py::test_f16_emulation_floor).  The router:
# f32 throughout, its logits within ROUTER_BOUND of float64; the engine's route equals the oracle's whenever the
# oracle's logit margin exceeds twice the bound plus the f16 trunk's effect on the logits (MARGIN).
FWD_GATE, ROUTER_BOUND, MARGIN = 1.5e-3, 1e-5, 0.05


def _engine(sd, cfg, h, w, processor=None):
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine(cfg, h, w, family="zoedepth", processor=processor)
    e.load_state_dict(sd)
    return e


def _force(sd, route, margin=50.0):
    sd = dict(sd)
    b = torch.zeros(2)
    b[route] = margin
    sd[ZO.M + "mlp_classifier.linear2.bias"] = b
    return sd


@pytest.fixture(scope="module")
def multi():
    return ZO.random_model(multi=True, seed=3)


@pytest.fixture(scope="module")
def single():
    return ZO.random_model(multi=False, seed=4)


def _forward_err(sd, cfg, h, w, seed, route=None):
    torch.manual_seed(seed)
    px = torch.randn(3, h, w)
    with torch.no_grad():
        ref, parts = ZO.forward(sd, cfg, px, route=route, return_parts=True)
    e = _engine(sd, cfg, h, w)
    out = e.forward(px.numpy())
    logits = e.get_buffer("z.logits", (2,), np.float32) if len(cfg["bins"]) > 1 else None
    e.close()
    ref = ref.numpy()
    return float(np.abs(out - ref).max() / (ref.max() - ref.min())), parts, logits


@pytest.mark.parametrize("route,hw", [(0, (64, 96)), (1, (96, 64)), (0, (128, 192)), (1, (384, 672))])
def test_forward_matches_oracle_two_configurations(multi, route, hw):
    sd, cfg = multi
    sd = _force(sd, route)
    err, parts, logits = _forward_err(sd, cfg, *hw, seed=7, route=route)
    print(f"ZoeDepth small route {route} {hw}: max-abs error / range {err:.3e}, logits {logits}")
    assert int(logits[1] > logits[0]) == route
    assert err <= FWD_GATE


@pytest.mark.parametrize("hw", [(64, 64), (96, 160)])
def test_forward_matches_oracle_single_configuration(single, hw):
    sd, cfg = single
    err, _, _ = _forward_err(sd, cfg, *hw, seed=9)
    print(f"ZoeDepth single-config small {hw}: max-abs error / range {err:.3e}")
    assert err <= FWD_GATE


@pytest.mark.parametrize("route", [0, 1])
def test_forward_matches_oracle_large_1080p_size(route):
    """BEiT-L/16 ZoeDepth at 384 x 672, the processed size of a 1920 x 1080 frame (1009 tokens), each route forced by
    the classifier's bias."""
    sd, cfg = ZO.random_model(multi=True, small=False, seed=1)
    err, _, logits = _forward_err(_force(sd, route), cfg, 384, 672, seed=11, route=route)
    print(f"ZoeDepth BEiT-L 384x672 route {route}: max-abs error / range {err:.3e}")
    assert int(logits[1] > logits[0]) == route
    assert err <= FWD_GATE


def test_route_equals_oracle_when_the_margin_allows(multi):
    """The classifier's last layer is scaled so that the random inputs give logit margins on both sides of MARGIN."""
    sd, cfg = multi
    sd = dict(sd)
    w = ZO.M + "mlp_classifier.linear2.weight"
    sd[w] = sd[w] * 300.0
    checked = 0
    for seed in range(6):
        torch.manual_seed(100 + seed)
        px = torch.randn(3, 64, 96) * (0.5 + seed)
        with torch.no_grad():
            _, parts = ZO.forward(sd, cfg, px, return_parts=True)
        e = _engine(sd, cfg, 64, 96)
        e.forward(px.numpy())
        lg = e.get_buffer("z.logits", (2,), np.float32)
        e.close()
        ref = parts["logits"].numpy()
        if abs(ref[1] - ref[0]) > MARGIN:
            assert int(lg[1] > lg[0]) == parts["route"]
            checked += 1
    print(f"routes compared: {checked} of 6")
    assert checked >= 3


# ---------------------------------------------------------------------------------------------------------------------
# the kernels on their own, through vd3d_zoe_kernel
# ---------------------------------------------------------------------------------------------------------------------
def _put(e, name, arr):
    arr = np.ascontiguousarray(arr)
    e.check(e.lib.vd3d_depth_set_tensor(e.h, name.encode(), arr.ctypes.data, arr.nbytes))


def _run(e, op, dims):
    e.check(e.lib.vd3d_zoe_kernel(e.h, op, (C.c_int32 * len(dims))(*dims)))


@pytest.fixture(scope="module")
def hook(multi):
    sd, cfg = multi
    e = _engine(sd, cfg, 64, 96)
    yield e
    e.close()


@pytest.mark.parametrize("w,h", [(1920, 1080), (1080, 1920), (333, 97), (16, 16)])
def test_preprocess_matches_transformers(hook, w, h):
    from transformers import ZoeDepthImageProcessor
    proc = ZoeDepthImageProcessor(ensure_multiple_of=32, keep_aspect_ratio=True, size={"height": 384, "width": 512})
    rng = np.random.default_rng(w + 3 * h)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    ref = proc(images=img, return_tensors="pt")["pixel_values"][0].numpy()
    OH, OW = ref.shape[1:]
    _put(hook, "t.img", img)
    _run(hook, 0, [h, w, OH, OW, 0])
    out = hook.get_buffer("t.out", (3, OH, OW), np.float32)
    err = float(np.abs(out - ref).max())
    print(f"preprocess {w}x{h} -> {OW}x{OH}: max abs {err:.3e}")
    assert err <= 2e-6


def test_router_logits_against_float64(multi, hook):
    sd, cfg = multi
    from visiondepth3d_b200.depth_weights import prepare_zoedepth, zoedepth_position_code
    F_ = cfg["fusion"]
    n = 12 * 21  # the bottleneck of a 1080p frame
    rng = np.random.default_rng(0)
    x = rng.standard_normal((n, F_)).astype(np.float32)
    packed = prepare_zoedepth(sd, cfg, 64, 96)
    _put(hook, "t.x", x)
    _put(hook, "t.w", packed["z.router"])
    _put(hook, "t.pe", zoedepth_position_code(n + 1).numpy())
    _run(hook, 1, [n, F_])
    got = hook.get_buffer("t.out", (2,), np.float32)
    sd64 = {k: v.double() for k, v in sd.items() if v.is_floating_point()}
    xm = torch.from_numpy(x).double().t().reshape(1, F_, 12, 21)
    with torch.no_grad():
        # the oracle's router in float64 (the sinusoid in f32 as transformers builds it, then widened)
        ref = HZ.router64(sd64, xm).numpy()
    err = float(np.abs(got - ref).max())
    print(f"router logits {got} vs float64 {ref}: max abs {err:.3e}")
    assert err <= ROUTER_BOUND


@pytest.mark.parametrize("seed_stage,route", [(True, 1), (False, 0)])
def test_attractor_against_float64(hook, seed_stage, route):
    """Half of the attractors sit on bins (zero conv2 rows, Softplus(b) equal to a bin), and pairs of bins coincide."""
    rng = np.random.default_rng(5 + route)
    nc, na, E, K = 2, 16, 128, 64
    H, W, Hp, Wp = 24, 42, 12, 21
    hid = np.maximum(rng.standard_normal((H * W, nc * E)), 0).astype(np.float16)
    w2 = (rng.standard_normal((nc, na, E)) * 0.05).astype(np.float32)
    prev_nat = (rng.random((Hp * Wp, K)) * 4).astype(np.float32)
    prev_nat[:, 1::2] = prev_nat[:, 0::2]  # coincident bins
    b2 = (rng.standard_normal((nc, na)) * 0.5).astype(np.float32)
    w2[:, ::2] = 0.0
    target = float(prev_nat[0, 0]) + 1e-6
    b2[:, ::2] = np.float32(np.log(np.expm1(target)))  # attractors a hair away from bin 0 of pixel 0
    if seed_stage:  # prev holds the raw conv2 of both configurations; Softplus first
        raw = np.log(np.expm1(np.maximum(prev_nat, 1e-3))).astype(np.float32)
        prev = np.zeros((Hp * Wp, nc * K), np.float32)
        prev[:, route * K:(route + 1) * K] = raw
        nat64 = np.log1p(np.exp(raw.astype(np.float64)))
    else:
        prev = prev_nat
        nat64 = prev_nat.astype(np.float64)
    _put(hook, "t.hid", hid)
    _put(hook, "t.w2", w2)
    _put(hook, "t.b2", b2)
    _put(hook, "t.prev", prev)
    _run(hook, 2, [H, W, Hp, Wp, nc, route, na, int(seed_stage)])
    got = hook.get_buffer("t.out", (H * W, K), np.float32)
    ref, _, _ = HZ.attractor(hid[:, route * E:(route + 1) * E], w2[route], b2[route], prev[:, route * K:(route + 1) * K]
                             if seed_stage else prev, Hp, Wp, H, W, prev_softplus=seed_stage)
    err = float(np.abs(got - ref).max() / (np.abs(ref).max()))
    print(f"attractor (seed {seed_stage}, route {route}): max abs / max {err:.3e}")
    assert err <= 2e-6


@pytest.mark.parametrize("cat,hid,route,p_end", [(0, 40, 0, 1), (0, 40, 1, 0), (1, 80, 0, 1)])
def test_log_binomial_against_float64(hook, cat, hid, route, p_end):
    """t pinned at min_temp (0.0212: the logits reach ~ -3e4), p driven to 1 - 1e-4 or to 1e-4 by the MLP's bias."""
    rng = np.random.default_rng(11 + cat + route)
    nc, E, K = 2, 128, 64
    H, W, He, We = 48, 84, 24, 42
    cin = 32 + cat + E
    act = np.maximum(rng.standard_normal((H * W, 32)), 0).astype(np.float16)
    emb = rng.standard_normal((He * We, E)).astype(np.float16)
    bins = np.sort(rng.random((He * We, K)) * 10, axis=1).astype(np.float32)
    w3 = (rng.standard_normal(32) * 0.3).astype(np.float32)
    b3 = np.array([0.1], np.float32)
    blocks = []
    for c in range(nc):
        w1 = (rng.standard_normal((cin, hid)) * 0.05).astype(np.float32)
        b1 = (rng.standard_normal(hid) * 0.1).astype(np.float32)
        w2 = (rng.standard_normal((4, hid)) * 0.05).astype(np.float32)
        pb = 12.0 if (c == route) == bool(p_end) else -12.0
        b2 = np.array([pb, -pb, 0.0, 0.0], np.float32)
        blocks.append((w1, b1, w2, b2))
    lb = np.concatenate([np.concatenate([w1.ravel(), b1, w2.ravel(), b2]) for w1, b1, w2, b2 in blocks]).astype(np.float32)
    tmin = 0.0212
    temp = np.array([tmin, tmin], np.float32)  # t = min_temp whatever the MLP says
    for n, v in (("t.act", act), ("t.emb", emb), ("t.bins", bins), ("t.lb", lb), ("t.temp", temp), ("t.w3", w3),
                 ("t.b3", b3)):
        _put(hook, n, v)
    _run(hook, 3, [H, W, He, We, nc, route, cat, hid])
    got = hook.get_buffer("t.out", (H * W,), np.float32)
    ref = HZ.log_binomial(act, emb, bins, He, We, H, W, HZ.logbinom_unpack(lb, nc, cin, hid, route), tmin, tmin,
                          w3 if cat else None, b3 if cat else None)
    err = float(np.abs(got - ref).max() / 10.0)
    print(f"log-binomial (cat {cat}, hid {hid}, route {route}, p -> {p_end}): max abs / bin span {err:.3e}")
    assert err <= 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# batches route per image
# ---------------------------------------------------------------------------------------------------------------------
def test_batch_with_mixed_routes_equals_single_forwards(multi):
    """Frames of one 1080p clip whose routes differ (the classifier's bias puts the split between them) give the same
    bytes in a batch of four as alone."""
    from visiondepth3d_b200.synth import synth_frame
    sd, cfg = multi
    e = _engine(sd, cfg, 384, 672)
    frames = [synth_frame(i, 1920, 1080, k)[0] for i, k in
              ((1, "natural"), (2, "noise"), (3, "smooth"), (4, "natural"), (5, "noise"), (6, "smooth"))]
    diffs = []
    for f in frames:
        e.infer(f)
        lg = e.get_buffer("z.logits", (2,), np.float32)
        diffs.append(float(lg[1] - lg[0]))
    order = np.argsort(diffs)
    lo, hi = order[len(order) // 2 - 1], order[len(order) // 2]
    shift = -(diffs[lo] + diffs[hi]) / 2  # the split between the two middle frames
    sd2 = dict(sd)
    b = sd[ZO.M + "mlp_classifier.linear2.bias"].clone()
    b[1] += shift
    sd2[ZO.M + "mlp_classifier.linear2.bias"] = b
    e.load_state_dict(sd2)
    pick = [frames[i] for i in (order[0], order[-1], lo, hi)]
    routes, singles = [], []
    for f in pick:
        singles.append(e.infer(f))
        lg = e.get_buffer("z.logits", (2,), np.float32)
        routes.append(int(lg[1] > lg[0]))
    assert sorted(routes) == [0, 0, 1, 1], (routes, diffs)
    batch = e.infer_batch(pick)
    for (d32, d8), (s32, s8) in zip(batch, singles):
        assert np.array_equal(d32, s32) and np.array_equal(d8, s8)
    e.close()


def test_post_process_crops_the_padding(multi):
    """infer's depth at the frame's size is the bicubic resize to the padded size, cropped (the oracle's post_process
    of the engine's own processed-size depth)."""
    sd, cfg = multi
    from visiondepth3d_b200.synth import synth_frame
    e = _engine(sd, cfg, 384, 672)
    f = synth_frame(7, 1920, 1080, "natural")[0]
    d32, d8 = e.infer(f)
    proc = e.get_buffer("depth", (384, 672), np.float32)
    ref = ZO.post_process(torch.from_numpy(proc), (1080, 1920)).numpy()
    err = float(np.abs(d32 - ref).max() / (ref.max() - ref.min()))
    assert err <= 1e-5, err
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
# the family's argument checks
# ---------------------------------------------------------------------------------------------------------------------
def test_set_zoe_arguments(multi):
    sd, cfg = multi
    e = _engine(sd, cfg, 64, 96)
    lib = e.lib
    f2 = (C.c_float * 2)(1e-3, 1e-3)
    g2 = (C.c_float * 2)(10.0, 80.0)

    def call(nc=2, nb=64, tmin=0.0212, tmax=50.0, att=(16, 16, 16, 16), cat=0, lo=f2, hi=g2, h=e.h):
        return lib.vd3d_depth_set_zoe(h, nc, nb, lo, hi, tmin, tmax, (C.c_int32 * 4)(*att), cat)
    assert call() == 0
    ERR_ARG = -2
    for kw in (dict(nc=3), dict(nc=0), dict(nb=32), dict(tmin=0.0), dict(tmax=0.01), dict(att=(16, 0, 4, 1)),
               dict(att=(17, 8, 4, 1)), dict(cat=2), dict(hi=(C.c_float * 2)(1e-4, 80.0))):
        assert call(**kw) == ERR_ARG, kw
    e.close()
    from visiondepth3d_b200.depth_engine import DepthEngine
    beit = DepthEngine({**cfg, "image_size": 64}, 64, 64, family="dpt-beit")
    assert call(h=beit.h) == ERR_ARG  # another family
    beit.close()


def test_clip_depth_and_tiled_depth_refuse_zoedepth(multi):
    """The joined depth -> stereo path and the tiled path serve Depth-Anything-V2 engines only: VD3D_ERR_UNSUPPORTED."""
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R3
    from visiondepth3d_b200.render_depth import _plan_for
    from visiondepth3d_b200.synth import synth_frame
    sd, cfg = multi
    e = _engine(sd, cfg, 64, 96)
    w, h = 320, 180
    rp = R3.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, "Half-SBS", 16 / 9, 0.0, 10.0, 9, True, True)
    frames = [synth_frame(i, w, h, "smooth")[0] for i in range(2)]
    outs = [np.empty((h, w, 3), np.uint8) for _ in frames]
    vp = C.c_void_p
    ctx = e.ctx
    assert ctx.lib.vd3d_render_clip_depth(ctx.h, e.h, 2, (vp * 2)(*[f.ctypes.data for f in frames]), h, w,
                                          C.byref(rp), (vp * 2)(*[o.ctypes.data for o in outs]), _lib.MEM_HOST) == -3
    plan = _plan_for(60, 50, 96, 16)
    frame = np.zeros((50, 60, 3), np.uint8)
    u8 = np.empty((50, 60), np.uint8)
    rc = ctx.lib.vd3d_depth_tiled(ctx.h, (vp * 1)(e.h), 1, 1, (vp * 1)(frame.ctypes.data), 50, 60, 96, 16, plan.tiles,
                                  len(plan.rects), plan.weight_ptrs, 0, 50, 60, (vp * 1)(u8.ctypes.data), None, None,
                                  _lib.MEM_HOST)
    assert rc == -3
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
# the drivers of render_depth on a save_pretrained folder (BEiT-L/16 ZoeDepth, the menu's configuration)
# ---------------------------------------------------------------------------------------------------------------------
PREPROC = dict(do_resize=True, do_rescale=True, do_normalize=True, do_pad=True, keep_aspect_ratio=True,
               ensure_multiple_of=32, size={"height": 384, "width": 512}, resample=2, image_mean=[0.5] * 3,
               image_std=[0.5] * 3)


class Var:
    def __init__(self, v):
        self.v = v

    def get(self):
        return self.v


@pytest.fixture(scope="module")
def zoe(tmp_path_factory):
    import json
    from visiondepth3d_b200 import render_depth as RD
    sd, _ = ZO.random_model(multi=True, small=False, seed=2)
    model = ZO.hf_model(sd, small=False)
    root = tmp_path_factory.mktemp("w")
    folder = root / "weights" / "Intel_zoedepth-nyu-kitti"
    model.save_pretrained(str(folder))
    with open(folder / "preprocessor_config.json", "w") as f:
        json.dump(dict(PREPROC, image_processor_type="ZoeDepthImageProcessor"), f)
    old = RD.local_model_dir
    RD.local_model_dir = str(root / "weights")
    RD.update_pipeline("ZoeDepth", None, None, None).join()
    yield RD, model
    RD.local_model_dir = old


def test_process_image_matches_transformers_pipeline(zoe, tmp_path):
    """A 1920 x 1080 image through process_image against transformers' pipeline("depth-estimation") on the same folder
    on the CPU (ZoeDepth's post-process: the padded resize, the crop), then convert_depth_to_grayscale."""
    from PIL import Image
    from transformers import ZoeDepthImageProcessor, pipeline
    from visiondepth3d_b200.synth import synth_frame
    RD, model = zoe
    assert RD._arch == "zoedepth-nyu-kitti" and RD.model_processed_size(1920, 1080) == (384, 672)
    fr, _ = synth_frame(5, 1920, 1080, "natural")
    img = Image.fromarray(fr[..., ::-1].copy())
    src = tmp_path / "in.png"
    img.save(src)
    RD.process_image(str(src), Var("default"), Var(False), Var(str(tmp_path / "o")), Var("Original"), None, None, None,
                     None)
    got = np.array(Image.open(tmp_path / "o" / "in_depth.png"))
    assert got.shape == (1080, 1920)
    proc = ZoeDepthImageProcessor(**{k: v for k, v in PREPROC.items()})
    pipe = pipeline("depth-estimation", model=model, image_processor=proc, device="cpu")
    with torch.no_grad():
        d = pipe(img)["predicted_depth"]
    want = RD.convert_depth_to_grayscale(d)
    diff = np.abs(got.astype(int) - want.astype(int))
    print("ZoeDepth process_image vs transformers pipeline: max LSB", int(diff.max()), "share > 0",
          float((diff > 0).mean()))
    assert diff.max() <= 1


def test_folder_of_mixed_sizes_and_a_depth_video_clip(zoe, tmp_path):
    import cv2
    from PIL import Image
    from tests import letterbox_oracle as L
    from tests.test_letterbox_cpu import _Cap
    RD, _ = zoe
    src = tmp_path / "in"
    src.mkdir()
    rng = np.random.default_rng(2)
    sizes = [(1280, 720), (720, 1280), (640, 360)]
    for k, (w, h) in enumerate(sizes):
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(src / f"im{k}.png")
    out = tmp_path / "out"
    RD.process_images_in_folder(str(src), 8, str(out), "Original", None, None, None, False)
    for k, (w, h) in enumerate(sizes):
        got = np.array(Image.open(out / f"im{k}_depth.png"))
        want = RD.convert_depth_to_grayscale(RD.hf_batch_safe_pipe([Image.open(src / f"im{k}.png")])[0]["predicted_depth"])
        assert got.shape == (h, w) and np.abs(got.astype(int) - want.astype(int)).max() <= 1
    frames = L.track_frames()[:6]
    h, w = frames[0].shape[:2]
    got = list(RD.iter_depth_frames(_Cap(frames, 2), w, h, False, None, batch_size=4))
    assert len(got) == len(frames)
    for f, g in zip(frames, got):
        assert np.abs(g.astype(int) - RD.depth_u8_from_frame(f).astype(int)).max() <= 1
    clip = str(tmp_path / "clip.avi")
    wr = cv2.VideoWriter(clip, cv2.VideoWriter_fourcc(*"MJPG"), 24.0, (w, h))
    for f in frames:
        wr.write(f)
    wr.release()
    assert RD.depth_video_from_video(clip, str(tmp_path / "depth.avi")) == len(frames)
