"""CPU restatement of the RRDBNet upscalers (ESRGAN, Wang et al. 2018: the generator of Real-ESRGAN's RealESRGAN_x4plus
and of BSRGAN x4 / x2) and of run_esrgan's chain around them.  TEST INFRASTRUCTURE ONLY.

The reference ships these networks as ONNX files only (VisionDepth3D.py:1094-1100); the graph is restated from the
published architecture on the basicsr naming (`conv_first`, `body.{i}.rdb{j}.conv{k}`, `conv_body`, `conv_up1/2`,
`conv_hr`, `conv_last`):
    feat = conv_first(x);  trunk = nb x RRDB(feat);  feat = feat + conv_body(trunk)
    per x2 of the scale: feat = lrelu(conv_up(nearest x2(feat)));  out = conv_last(lrelu(conv_hr(feat)))
    RDB: x1..x4 = lrelu(conv_k(cat(x, x1, ..))), x5 = conv5(cat(x, x1..x4)), returns x + 0.2 x5
    RRDB: x + 0.2 rdb3(rdb2(rdb1(x)));  lrelu = LeakyReLU(0.2).
rrdb_forward is that graph in fp32.  rrdb_forward_f16 is the same graph with the weights and every activation rounded
to f16 where libvd3d stores them (network input, each conv output after its epilogue: the dense features after the
LeakyReLU, the RDB output x + 0.2 x5, the RRDB output written by the third RDB's last conv without rounding the RDB
output in between, the trunk sum, each up-conv and conv_hr output); the arithmetic stays fp32 and conv_last's output
is not rounded.  It is the gate for the kernels.
"""
import numpy as np

from oracle.sr import blend_images, postprocess_esr, preprocess_esr, resize_cubic_bgr


def _t(sd):
    """basicsr-named float32 torch tensors of a state dict in either naming (the key mapping restated here)."""
    import re
    import torch
    ren = [(r"^RRDB_trunk\.(\d+)\.RDB(\d)\.conv(\d)\.", r"body.\1.rdb\2.conv\3."), (r"^trunk_conv\.", "conv_body."),
           (r"^upconv1\.", "conv_up1."), (r"^upconv2\.", "conv_up2."), (r"^HRconv\.", "conv_hr.")]
    out = {}
    for k, v in sd.items():
        for a, b in ren:
            k = re.sub(a, b, k)
        out[k] = torch.as_tensor(np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, np.float32))
    return out


def _graph(sd, x, q, qw):
    import torch
    import torch.nn.functional as F
    nb = len({k.split(".")[1] for k in sd if k.startswith("body.")})

    def conv(name, t):
        return F.conv2d(t, qw(sd[name + ".weight"]), sd[name + ".bias"], padding=1)

    def lrelu(t):
        return F.leaky_relu(t, 0.2)

    def rdb(x, pre, rrdb_in=None):
        feats = [x]
        for k in range(1, 5):
            feats.append(q(lrelu(conv(f"{pre}.conv{k}", torch.cat(feats, 1)))))
        x5 = conv(f"{pre}.conv5", torch.cat(feats, 1))
        if rrdb_in is None:
            return q(x + 0.2 * x5)
        return q(rrdb_in + 0.2 * (x + 0.2 * x5))  # the RRDB residual in the same epilogue: one rounding

    with torch.no_grad():
        x = q(x)
        feat = q(conv("conv_first", x))
        t = feat
        for i in range(nb):
            r = rdb(t, f"body.{i}.rdb1")
            r = rdb(r, f"body.{i}.rdb2")
            t = rdb(r, f"body.{i}.rdb3", rrdb_in=t)
        feat = q(feat + conv("conv_body", t))
        for u in (1, 2):
            if f"conv_up{u}.weight" in sd:
                feat = q(lrelu(conv(f"conv_up{u}", F.interpolate(feat, scale_factor=2, mode="nearest"))))
        return conv("conv_last", q(lrelu(conv("conv_hr", feat))))


def rrdb_forward(sd, x):
    """x f32 [1,3,h,w] RGB in 0..1 -> f32 [1,3,s h,s w] (RRDBNet.forward in fp32)."""
    ident = lambda t: t
    return _graph(_t(sd), x, ident, ident)


def rrdb_forward_f16(sd, x):
    """rrdb_forward with the weights and the stored activations rounded to f16 (see the module docstring)."""
    import torch
    q = lambda t: t.to(torch.float16).to(torch.float32)
    return _graph(_t(sd), x, q, q)


def net_scale(sd):
    return 4 if any(k.startswith(("conv_up2.", "upconv2.")) for k in sd) else 2


def upscale(sd, frame_bgr, forward=rrdb_forward_f16):
    """preprocess_esr -> network -> postprocess_esr: BGR u8 [h,w,3] -> BGR u8 [s h, s w, 3]."""
    import torch
    return postprocess_esr(forward(sd, torch.from_numpy(preprocess_esr(frame_bgr))).numpy())


def run_esrgan(sd, frame_bgr, blend_mode="OFF", input_res_pct=100, model_name="RealESR_Gx4_fp16", target_size=None,
               network=None):
    """core/merged_pipeline.py:240-267 without tiling on an RRDBNet: optional input resize (INTER_AREA below 100 %,
    INTER_CUBIC above), network (net scale s; `network` maps the BGR u8 input to the BGR u8 output, default
    upscale(sd, .)), INTER_CUBIC to scale x the network input with scale = 2 if "x2" in model_name.lower() else 4 (a
    copy when that is s), back to the original size, optionally to target_size, blend_images."""
    from oracle.dibr import resize_area
    original = frame_bgr
    frame = frame_bgr
    if input_res_pct != 100:
        h, w = frame.shape[:2]
        nw, nh = int(w * input_res_pct / 100), int(h * input_res_pct / 100)
        frame = resize_area(frame, nw, nh) if input_res_pct < 100 else resize_cubic_bgr(frame, nw, nh)
    up = network(frame) if network is not None else upscale(sd, frame)
    scale = 2 if "x2" in model_name.lower() else 4
    up = resize_cubic_bgr(up, frame.shape[1] * scale, frame.shape[0] * scale)
    up = resize_cubic_bgr(up, original.shape[1], original.shape[0])
    if target_size:
        up = resize_cubic_bgr(up, target_size[0], target_size[1])
    return blend_images(original, up, blend_mode)
