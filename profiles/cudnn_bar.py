"""The GPU library bar (SURVEY.md 8d): what the reference's own call chain -- nn.SpatialUpSamplingNearest(2) ->
cudnn.SpatialConvolution 5x5 (models.lua:63-64, :68-69) -- costs with today's cuDNN through PyTorch, at the G.C1 / G.C2
shapes of BASELINE configs[1] (batch 256), forward + input gradient + weight gradient, CUDA-event timed.
Measurement infrastructure only (PyTorch is not part of the product).  fp32 = TF32 disabled (the parity-equivalent
setting); "tf32" = cuDNN allowed to use TF32 tensor cores (1e-3 relative error: would fail the 1e-4 bar).

usage:  python profiles/cudnn_bar.py > cudnn_bar.jsonl"""
import json

import torch
import torch.nn.functional as F


def timed(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def layer(name, B, Cin, Hlow, Cout, k, allow_tf32, channels_last):
    torch.backends.cudnn.allow_tf32 = allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = allow_tf32
    torch.backends.cudnn.benchmark = True
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    low = torch.randn(B, Cin, Hlow, Hlow, device="cuda")
    w = torch.randn(Cout, Cin, k, k, device="cuda").contiguous(memory_format=fmt)
    bias = torch.randn(Cout, device="cuda")
    up = F.interpolate(low, scale_factor=2, mode="nearest").contiguous(memory_format=fmt)
    dy = torch.randn(B, Cout, 2 * Hlow, 2 * Hlow, device="cuda").contiguous(memory_format=fmt)
    t_up = timed(lambda: F.interpolate(low, scale_factor=2, mode="nearest"))
    t_fwd = timed(lambda: F.conv2d(up, w, bias, padding=k // 2))
    t_dx = timed(lambda: torch.nn.grad.conv2d_input(up.shape, w, dy, padding=k // 2))
    t_dw = timed(lambda: torch.nn.grad.conv2d_weight(up, w.shape, dy, padding=k // 2))
    flops = 2.0 * Cout * Cin * k * k * (2 * Hlow) ** 2 * B
    return {"layer": name, "math": "tf32" if allow_tf32 else "fp32", "layout": "NHWC" if channels_last else "NCHW",
            "upsample_ms": round(t_up, 4), "fwd_ms": round(t_fwd, 4), "dgrad_ms": round(t_dx, 4), "wgrad_ms": round(t_dw, 4),
            "fwd_tflops": round(flops / t_fwd / 1e9, 1), "cudnn": torch.backends.cudnn.version(), "torch": torch.__version__}


if __name__ == "__main__":
    for tf32 in (False, True):
        for cl in (False, True):
            print(json.dumps(layer("G.C2 up2+5x5 256->128 @32x32", 256, 256, 16, 128, 5, tf32, cl)), flush=True)
            print(json.dumps(layer("G.C1 up2+5x5 128->256 @16x16", 256, 128, 8, 256, 5, tf32, cl)), flush=True)
