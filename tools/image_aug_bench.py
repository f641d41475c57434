"""The camera augmentation of one nuScenes sample on the device: six 1600x900 uint8 images through ImageAug3D +
ImageNormalize (resize, crop, flip, rotate, normalise) to [6, 3, 256, 704] fp32.

    python tools/image_aug_bench.py OUT_DIR [--window 1.0] [--rounds 3] [--pillow-images 12]

At B = 1 and 4, with seeded training draws of the nuScenes config (resize 0.38-0.55, rotation +-5.4 deg, flip):
  eager_host_draws   image_aug with host draws (pinned staging, one asynchronous copy, three launches)
  eager_device_draws image_aug_batched with the draws already on the device
  graph              image_aug_batched captured as a CUDA graph and replayed
Each time is the median over --rounds alternating rounds of the mean CUDA-event time over a window of at least
--window seconds, reported per sample.  Also: the device time per kernel from a torch.profiler run after the timing,
the shape-derived HBM floor per sample (every uint8 input byte read once, every fp32 output byte written once, at the
data sheet's 3.35 TB/s) and the timed figure as a share of it, and Pillow + torchvision's host time per image for the
same draws (one core).  The card name and power limit are read in the same run.  Writes OUT_DIR/image_aug_bench.json.
Needs a CUDA device."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bevfusion_b200.image_aug import ImageAug3D, image_aug, image_aug_batched, pack_draw  # noqa: E402
from encoder_fp16_bench import card_info, graph_of, kernel_us, timed_ms  # noqa: E402

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
H, W, N, FH, FW = 900, 1600, 6, 256, 704
HBM_BYTES_PER_S = 3.35e12
CFG = dict(final_dim=(FH, FW), resize_lim=(0.38, 0.55), bot_pct_lim=(0.0, 0.0), rot_lim=(-5.4, 5.4), rand_flip=True,
           is_train=True)


def images(B, seed):
    rng = np.random.RandomState(seed)
    return torch.from_numpy(rng.randint(0, 256, (B, N, H, W, 3), dtype=np.uint8))


def pillow_ms_per_image(imgs, draws, count):
    try:
        import torchvision.transforms.functional as TF
        from PIL import Image
    except ImportError:
        return None
    times = []
    for i in range(count):
        img = imgs[i % imgs.shape[0]]
        _, dims, crop, flip, rotate = draws[i % len(draws)]
        t = time.perf_counter()
        im = Image.fromarray(img).resize(dims).crop(crop)
        if flip:
            im = im.transpose(Image.FLIP_LEFT_RIGHT)
        TF.normalize(TF.to_tensor(im.rotate(rotate)), MEAN, STD)
        times.append((time.perf_counter() - t) * 1e3)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pillow-images", type=int, default=12)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    dev = torch.device("cuda")
    aug = ImageAug3D(**CFG, rng=np.random.RandomState(0))
    min_resize = aug.min_resize((W, H))
    floor_us = (N * H * W * 3 + N * 3 * FH * FW * 4) / HBM_BYTES_PER_S * 1e6
    result = {"card": card_info(), "shape": "6 x 1600x900 uint8 -> 6 x 3 x 256x704 fp32 per sample",
              "hbm_floor_us_per_sample": floor_us, "rows": []}
    for B in (1, 4):
        x = images(B, B).to(dev)
        draws = [aug.draws((W, H), N) for _ in range(B)]
        dd = torch.tensor([[pack_draw(*d) for d in s] for s in draws], dtype=torch.float64, device=dev)
        fns = {"eager_host_draws": lambda: image_aug(x, draws, MEAN, STD),
               "eager_device_draws": lambda: image_aug_batched(x, dd, (FH, FW), MEAN, STD, min_resize)}
        g, _ = graph_of(lambda: image_aug_batched(x, dd, (FH, FW), MEAN, STD, min_resize))
        fns["graph"] = g.replay
        for fn in fns.values():
            fn()
        torch.cuda.synchronize()
        per = {k: [] for k in fns}
        for _ in range(args.rounds):
            for k, fn in fns.items():
                per[k].append(timed_ms(fn, args.window))
        row = {"B": B}
        for k, v in per.items():
            us = statistics.median(v) * 1e3 / B
            row[k + "_us_per_sample"] = us
        row["graph_share_of_hbm_floor"] = floor_us / row["graph_us_per_sample"]
        row["kernels"] = kernel_us(lambda: image_aug_batched(x, dd, (FH, FW), MEAN, STD, min_resize))
        result["rows"].append(row)
        print(json.dumps({k: v for k, v in row.items() if k != "kernels"}), flush=True)
    imgs = images(1, 99)[0].numpy()
    result["pillow_ms_per_image"] = pillow_ms_per_image(imgs, aug.draws((W, H), N), args.pillow_images)
    print(json.dumps({"card": result["card"], "hbm_floor_us_per_sample": floor_us,
                      "pillow_ms_per_image": result["pillow_ms_per_image"]}), flush=True)
    with open(os.path.join(args.out_dir, "image_aug_bench.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
