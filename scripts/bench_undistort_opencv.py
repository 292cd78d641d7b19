"""Frame staging from a RAW camera image with an OpenCV-model (radial-tangential) calibration, at 640x480 and 1280x1024:
(a) the host undistorts (cv2.remap through the CV_16SC2 maps when the cv2 module is importable, otherwise the tests' C
    restatement of cv::remap -- the output line says which) and the undistorted image goes through lsdgpu_frame_upload_u8,
(b) lsdgpu_frame_upload_distorted_u8: one H2D copy of the raw image, the remap feeds the pyramid kernel.
Per frame: device time (CUDA events on the context's stream around the upload call) and wall time (host clock around the
whole step, ending in a device synchronise), medians.  Prints one JSON line."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.getcwd())
import torch  # noqa: E402  (pinned host buffer for the raw image)

from lsd_slam_b200 import abi  # noqa: E402

TUM_FR1 = [517.3, 516.5, 318.6, 255.3, 0.2624, -0.9531, -0.0054, 0.0026]
try:
    import cv2
    HOST_REMAP = "cv2.remap (OpenCV %s, %d threads)" % (cv2.__version__, cv2.getNumThreads())

    def host_remap(raw, m1, m2):
        return cv2.remap(raw, m1, m2, cv2.INTER_LINEAR)
except ImportError:
    from tests import undistort_opencv_oracle as cvo
    HOST_REMAP = "C restatement of cv::remap (tests/native/undistort_opencv_oracle.c, one thread)"

    def host_remap(raw, m1, m2):
        return cvo.remap(raw, m1, m2)


def run(w, h, frames=200, warmup=20):
    s = w / 640.0
    calib = [TUM_FR1[0] * s, TUM_FR1[1] * s, TUM_FR1[2] * s, TUM_FR1[3] * h / 480.0] + TUM_FR1[4:]
    u = abi.UndistorterOpenCV(calib, (w, h), "crop", (w, h))
    ctx = abi.Context(w, h, u.getK(), max_frames=4)
    u.install(ctx)
    rng = np.random.default_rng(0)
    raw = torch.from_numpy(rng.integers(0, 256, (h, w)).astype(np.uint8)).pin_memory().numpy()
    assert np.array_equal(ctx.undistort(raw), host_remap(raw, u.map1, u.map2))
    res = {}
    for name in ("host_remap_then_upload", "fused_upload_distorted"):
        dev, wall = [], []
        for i in range(warmup + frames):
            t0 = time.perf_counter()
            if name == "host_remap_then_upload":
                img = host_remap(raw, u.map1, u.map2)
                ctx.timer_begin(0)
                ctx.upload(1, img)
            else:
                ctx.timer_begin(0)
                ctx.upload_distorted(1, raw)
            ctx.timer_end(0)
            ctx.synchronize()
            t1 = time.perf_counter()
            if i >= warmup:
                dev.append(ctx.timer_ms(0) * 1e3)
                wall.append((t1 - t0) * 1e6)
            ctx.release(1)
        res[name] = {"device_us": round(float(np.median(dev)), 2), "wall_us": round(float(np.median(wall)), 2)}
    ctx.close()
    return res


def main():
    out = {"workload": "raw u8 + OpenCV calibration (TUM fr1-like, crop) -> undistort -> pyramids + gradients + maxGradients",
           "host_remap": HOST_REMAP, "gpu": torch.cuda.get_device_name(0)}
    for w, h in ((640, 480), (1280, 1024)):
        out["%dx%d" % (w, h)] = run(w, h)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
