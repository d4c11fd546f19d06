"""CPU restatement of Real-ESRGAN x4 as the reference runs it (upsampling.py -> realesrgan's RealESRGANer.enhance with
half=True, tile=0 -> basicsr's RRDBNet), for tests only.

Neither basicsr nor realesrgan is vendored, so this is dependency knowledge, not pinned to reference source:
  u8 = round(img * 255); x = fp16(u8 / 255); y = RRDBNet(x); out = round(clamp(y, 0, 1) * 255)
RRDBNet (scale 4): conv_first; body = num_block x RRDB; feat += conv_body(body(feat));
lrelu(conv_up1(nearest x2)), lrelu(conv_up2(nearest x2)), conv_last(lrelu(conv_hr(.))); every conv 3x3, pad 1, bias.
RDB: x_k = lrelu(conv_k(cat(x, x_1..x_{k-1}))) for k = 1..4, x5 = conv5(cat(...)), returns 0.2 x5 + x;
RRDB: 0.2 rdb3(rdb2(rdb1(x))) + x.  LeakyReLU slope 0.2 everywhere.

`fp16_storage=True` rounds every conv output and every block output to fp16 (what a half-precision network stores
between layers), with fp32 arithmetic inside each op; it measures the error an fp16 implementation is expected to have.
"""
import numpy as np
import torch
import torch.nn.functional as F


def _conv(x, sd, name, fp16_storage):
    y = F.conv2d(x, sd[name + ".weight"], sd[name + ".bias"], padding=1)
    return y.half().float() if fp16_storage else y


def _lrelu(x):
    return F.leaky_relu(x, 0.2)


def _r(x, fp16_storage):
    return x.half().float() if fp16_storage else x


def rrdbnet(x, sd, num_block, fp16_storage=False):
    """x: float32 NCHW in [0, 1] -> float32 NCHW (4x), pre-clamp."""
    sd = {k: v.float() for k, v in sd.items()}
    feat = _conv(x, sd, "conv_first", fp16_storage)
    h = feat
    for i in range(num_block):
        inp = h
        for r in range(1, 4):
            p = f"body.{i}.rdb{r}."
            xs = [h]
            for k in range(1, 5):
                xs.append(_r(_lrelu(_conv(torch.cat(xs, 1), sd, p + f"conv{k}", fp16_storage)), fp16_storage))
            x5 = _conv(torch.cat(xs, 1), sd, p + "conv5", fp16_storage)
            h = _r(x5 * 0.2 + h, fp16_storage)
        h = _r(h * 0.2 + inp, fp16_storage)
    feat = _r(feat + _conv(h, sd, "conv_body", fp16_storage), fp16_storage)
    feat = _r(_lrelu(_conv(F.interpolate(feat, scale_factor=2, mode="nearest"), sd, "conv_up1", fp16_storage)), fp16_storage)
    feat = _r(_lrelu(_conv(F.interpolate(feat, scale_factor=2, mode="nearest"), sd, "conv_up2", fp16_storage)), fp16_storage)
    feat = _r(_lrelu(_conv(feat, sd, "conv_hr", fp16_storage)), fp16_storage)
    return _conv(feat, sd, "conv_last", fp16_storage)


def upsample_u8(frames_u8, sd, num_block, fp16_storage=False):
    """uint8 RGB [B, H, W, 3] (numpy) -> (uint8 [B, 4H, 4W, 3], float32 pre-clamp [B, 4H, 4W, 3])."""
    x = torch.from_numpy(np.ascontiguousarray(frames_u8)).float() / 255.0
    x = x.half().float().permute(0, 3, 1, 2).contiguous()
    with torch.no_grad():
        y = rrdbnet(x, sd, num_block, fp16_storage).permute(0, 2, 3, 1).contiguous()
    u8 = (y.clamp(0, 1) * 255.0).round().to(torch.uint8).numpy()
    return u8, y.numpy()
