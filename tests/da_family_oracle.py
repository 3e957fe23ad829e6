"""The Depth-Anything family for tests: random-init models of any spec (V1 taps, a metric head) and the fp32 forward
of oracle/depth.py with the metric head's max_depth * sigmoid in place of the final ReLU
(DepthAnythingDepthEstimationHead, transformers 5.5 models/depth_anything/modeling_depth_anything.py)."""
import torch
import torch.nn.functional as F

from oracle import depth as OD


def head_input(sd, cfg, px):
    """relu(conv2(...)) of the head, f32 [32, H, W]: what the last 1x1 conv of the head reads."""
    _, parts = OD.forward(sd, cfg, px, return_parts=True)
    IH, IW = px.shape[-2:]
    d = F.conv2d(parts["fused"][-1], sd["head.conv1.weight"], sd["head.conv1.bias"], padding=1)
    d = F.interpolate(d, (IH, IW), mode="bilinear", align_corners=True)
    return F.relu(F.conv2d(d, sd["head.conv2.weight"], sd["head.conv2.bias"], padding=1))[0]


def pre_activation(sd, h):
    """conv3 of the head on head_input: the value the last activation sees, [H, W]."""
    return F.conv2d(h[None], sd["head.conv3.weight"], sd["head.conv3.bias"])[0, 0]


def forward(sd, cfg, px, return_pre=False):
    """predicted_depth [H, W] of a Depth-Anything spec (depth_weights.da_spec): oracle.depth.forward for the relative
    head, max_depth * sigmoid(conv3) for the metric one.  return_pre: also the pre-activation."""
    if cfg.get("head", "relative") != "metric":
        out = OD.forward(sd, cfg, px)
        return (out, None) if return_pre else out
    s = pre_activation(sd, head_input(sd, cfg, px))
    out = torch.sigmoid(s) * cfg["max_depth"]
    return (out, s) if return_pre else out


def random_model(spec, seed=0, calib=None, span=4.0):
    """state dict of DepthAnythingForDepthEstimation(hf_config(spec)) at torch.manual_seed(seed), with the head's last
    1x1 conv made non-degenerate: PyTorch's symmetric init cancels it to ~1e-4 of its terms, which would put a metric
    model at max_depth / 2 everywhere.  Non-negative weights (like a trained head's); for a metric head, `calib`
    (pixel_values [3, h, w]) then sets the scale and bias so that the pre-sigmoid value spans [-span, span] there, so
    that both flat tails and the steep middle of the sigmoid are exercised."""
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200.depth_weights import da_spec, hf_config
    spec = da_spec(spec)
    torch.manual_seed(seed)
    sd = DepthAnythingForDepthEstimation(hf_config(spec)).eval().state_dict()
    sd["head.conv3.weight"] = sd["head.conv3.weight"].abs() + 0.02
    sd["head.conv3.bias"] = torch.zeros_like(sd["head.conv3.bias"])
    if spec["head"] == "metric":
        if calib is None:
            calib = torch.randn(3, 70, 98, generator=torch.Generator().manual_seed(seed + 1))
        with torch.no_grad():
            s = pre_activation(sd, head_input(sd, spec, calib))
        a = 2 * span / float(s.max() - s.min())
        sd["head.conv3.weight"] = sd["head.conv3.weight"] * a
        sd["head.conv3.bias"] = torch.tensor([-span - a * float(s.min())])
    return sd, spec
