"""Time the vignetteCalib optimiser kernels (plane step, vignette step, smoothing) on a synthetic device-resident problem:
n images of 1280x1024, 1000x1000 plane grid, smooth affine plane-to-image maps.  Prints one JSON line."""
import json, os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mono_dataset_code_b200 import api


def main():
    n = int(os.environ.get("VC_N", "256"))
    gw = gh = 1000
    wI, hI = 1280, 1024
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev); g.manual_seed(1)
    gy, gx = torch.meshgrid(torch.arange(gh, device=dev, dtype=torch.float32), torch.arange(gw, device=dev, dtype=torch.float32), indexing="ij")
    u, v = (gx / gw - 0.5).ravel(), (gy / gh - 0.5).ravel()
    p2x = torch.empty((n, gw * gh), dtype=torch.float32, device=dev)
    p2y = torch.empty_like(p2x)
    for i in range(n):
        ang, sc = 0.4 * np.sin(i), 500.0 + 250.0 * np.cos(0.37 * i)
        tx, ty = 640 + 150 * np.sin(0.11 * i), 512 + 120 * np.cos(0.23 * i)
        X = tx + sc * (np.cos(ang) * u - np.sin(ang) * v)
        Y = ty + sc * (np.sin(ang) * u + np.cos(ang) * v)
        bad = ~(((X + 0.5).int() > 1) & ((Y + 0.5).int() > 1) & ((X + 0.5).int() < wI - 2) & ((Y + 0.5).int() < hI - 2))
        X[bad] = float("nan"); Y[bad] = float("nan")
        p2x[i], p2y[i] = X, Y
    images = torch.rand((n, wI * hI), dtype=torch.float32, device=dev, generator=g) * 200 + 20
    plane = torch.full((gw * gh,), 100.0, dtype=torch.float32, device=dev)
    vig = torch.ones(wI * hI, dtype=torch.float32, device=dev)
    ctx = api.Context(None, None, 0)
    visible = float(torch.isfinite(p2x).float().mean().item())

    def timed(fn, reps=3):
        fn(); torch.cuda.synchronize(); t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / reps

    plane_ms = timed(lambda: ctx.vc_plane_step(images, p2x, p2y, gw, gh, wI, hI, vig, plane, 10000 * 10000))
    vig_ms = timed(lambda: ctx.vc_vignette_step(images, p2x, p2y, gw, gh, wI, hI, plane, vig, 10000 * 10000))
    smooth_ms = timed(lambda: ctx.vc_smooth(vig, wI, hI, 4))
    samples = n * gw * gh
    pc2, v2 = plane.clone(), vig.clone()
    ctx.vignette_calib(images, p2x, p2y, gw, gh, wI, hI, 1, 15, pc2, v2, True)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    ctx.vignette_calib(images, p2x, p2y, gw, gh, wI, hI, 4, 15, pc2, v2, True)
    torch.cuda.synchronize()
    loop_ms = (time.perf_counter() - t0) * 1e3 / 4      # incl. the one-off bounds pass and the final smoothing
    front = front_end(n, gw, gh, wI, hI, ctx, images, p2x, p2y, timed)
    print(json.dumps({"n": n, "plane_points": gw * gh, "visible_fraction": visible, "plane_step_ms": plane_ms, "vignette_step_ms": vig_ms,
                      "smooth4_ms": smooth_ms, "loop_ms_per_iteration": loop_ms, "plane_gsamples_per_s": samples / plane_ms / 1e6, "vignette_gsamples_per_s": samples / vig_ms / 1e6,
                      "map_bytes_gbs_plane": samples * 8 / plane_ms / 1e6, **front}), flush=True)


def front_end(n, gw, gh, wI, hI, ctx, images, p2x, p2y, timed):
    """The front end in front of the loop (main_vignetteCalib.cpp:266-301, :346-357) at the same scale: plane-to-image maps of n
    marker poses through a 1280x1024 'crop' camera (mdc_vc_plane_maps, written into p2x / p2y), and the image preparation
    (mdc_vc_prepare_images) of n calibration-pattern frames and of n dense-edge frames (a one-pixel checkerboard: every centre has
    candidate hits)."""
    import tempfile
    from mono_dataset_code_b200 import synthetic as S
    with tempfile.TemporaryDirectory() as tmp:
        fov = api.UndistorterFOV(S.write_dataset_dir(tmp, wI, hI, wI, hI, "crop")["camera"])
    Hs = []
    for i in range(n):
        ang, s = 0.4 * np.sin(i), 150.0 + 40.0 * np.cos(0.37 * i)
        Hs.append([s * np.cos(ang), -s * np.sin(ang), 640 + 150 * np.sin(0.11 * i), s * np.sin(ang), s * np.cos(ang), 512 + 120 * np.cos(0.23 * i),
                   2e-4 * np.cos(i), -1e-4 * np.sin(i), 1.0])
    maps_ms = timed(lambda: fov.vcPlaneMaps(Hs, gw, gh, p2x, p2y))
    dev = images.device
    yy, xx = torch.meshgrid(torch.arange(hI, device=dev), torch.arange(wI, device=dev), indexing="ij")
    pattern = (40.0 + 360.0 * (((xx // 64) + (yy // 64)) % 2)).float().reshape(1, -1)
    raw = (pattern + images[:, :] * 0.05).contiguous()                # pattern + noise: invalidation along the pattern's edges
    dense = (20.0 + 380.0 * ((xx + yy) % 2)).float().reshape(1, -1).expand(n, -1).contiguous()
    expo = np.linspace(0.5, 2.0, n).astype(np.float32)
    mean = float(expo.mean())
    out = torch.empty_like(raw)
    prep_ms = timed(lambda: ctx.vc_prepare_images(raw, wI, hI, expo, mean, 255, out=out))
    invalid = float(torch.isnan(out).float().mean().item())
    dense_ms = timed(lambda: ctx.vc_prepare_images(dense, wI, hI, expo, mean, 255, out=out))
    dense_invalid = float(torch.isnan(out).float().mean().item())
    return {"front_maps_ms": maps_ms, "front_maps_gpoints_per_s": n * gw * gh / maps_ms / 1e6, "front_maps_visible_fraction": float(torch.isfinite(p2x).float().mean().item()),
            "front_prepare_ms": prep_ms, "front_prepare_ms_per_image": prep_ms / n, "front_prepare_invalid_fraction": invalid,
            "front_prepare_dense_ms": dense_ms, "front_prepare_dense_ms_per_image": dense_ms / n, "front_prepare_dense_invalid_fraction": dense_invalid}


if __name__ == "__main__":
    main()
