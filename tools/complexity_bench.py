"""Times the match-complexity statistics: image_stats + jpeg_sizes (quality 90) on N device-resident 224 x 224 images,
with CUDA events (median of several calls after a warm-up), and reads the card's name and power limit in the same run.
When cv2 is importable it also times the reference's host loop (diff_retrieval.py:505-516, decode excluded) on a
sample and extrapolates it to N images -- labelled as an extrapolation.

    python tools/complexity_bench.py [--n 10000] [--reps 7] [--cpu-sample 200] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dcr_b200 import complexity, synthetic  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:   # the measurement stands without it, the record says why it is missing
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def time_gpu(imgs, reps):
    def once():
        complexity.image_stats(imgs)
        complexity.jpeg_sizes(imgs, 90)

    once()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        once()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def time_cpu_reference(imgs_np):
    import cv2
    from sklearn.metrics.cluster import entropy
    from oracle.complexity import grey_u8, tv_loss
    t0 = time.perf_counter()
    for rgb in imgs_np:
        entropy(grey_u8(rgb))
        cv2.imencode(".jpg", rgb, [int(cv2.IMWRITE_JPEG_QUALITY), 90])
        tv_loss(torch.from_numpy(rgb).permute(2, 0, 1).float().div(255) * 255)
    return (time.perf_counter() - t0) / len(imgs_np)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--cpu-sample", type=int, default=200)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("complexity_bench needs a CUDA device")
    base = synthetic.images(256, seed=1, size=224).cuda()
    imgs = base.repeat((args.n + 255) // 256, 1, 1, 1)[:args.n].contiguous()
    ms = time_gpu(imgs, args.reps)
    res = {"card": card(), "n_images": args.n, "size": 224, "gpu_ms_median": float(np.median(ms)),
           "gpu_ms_all": ms, "gpu_images_per_s": args.n / (np.median(ms) / 1e3)}
    try:
        import cv2  # noqa: F401
        sample = imgs[:args.cpu_sample].cpu().numpy()
        per = time_cpu_reference(sample)
        res["cpu_reference_ms_per_image"] = per * 1e3
        res["cpu_reference_s_for_n_extrapolated"] = per * args.n
    except ImportError:
        res["cpu_reference"] = "not measured (cv2 not importable)"
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
