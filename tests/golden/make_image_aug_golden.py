"""Generates tests/golden/image_aug_tiny.npz: Pillow + torchvision outputs of the camera augmentation for a handful
of draws, so that the GPU tests can check the device output without Pillow.

Each camera image goes through the reference pipeline's pixel steps as written in ImageAug3D.img_transform and
ImageNormalize (transforms_3d.py:125-131, 992-1006):

    TF.normalize(TF.to_tensor(img.resize(dims).crop(box)[.transpose(FLIP_LEFT_RIGHT)].rotate(deg)), mean, std)

Cases (two samples of six 45 x 80 cameras, 24 x 40 crops): downscale and upscale, crops inside and past every side
of the resized image, flips, and the rotations 0, +-5.4, a tiny angle, 90 (the affine path on a non-square crop),
180, -1e-20 (Pillow's scaling path) and 33.3 degrees.  Pillow's version is stored with the data.

Run:  python tests/golden/make_image_aug_golden.py"""
import os

import numpy as np
import PIL
import torchvision.transforms.functional as TF
from PIL import Image

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "image_aug_tiny.npz")
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
FINAL = (24, 40)
# resize, resize_dims, crop (x0, y0), flip, rotate
DRAWS = [[(0.6, (48, 27), (4, 3), False, 0.0), (0.55, (44, 24), (2, 0), True, 5.4),
          (0.7, (56, 31), (12, 6), False, -5.4), (1.3, (104, 58), (30, 20), True, 1e-7),
          (0.5, (40, 22), (-3, -2), False, 90.0), (2.0, (160, 90), (150, 80), True, 180.0)],
         [(0.45, (36, 20), (0, 0), True, -1e-20), (1.0, (80, 45), (20, 10), False, 33.3),
          (0.9, (72, 40), (30, 16), True, -2.25), (0.33, (26, 14), (-1, -5), False, 4.0),
          (1.75, (140, 78), (60, 40), False, -90.0), (0.62, (49, 27), (5, 3), True, 0.0)]]


def main():
    rng = np.random.RandomState(0)
    B, N = len(DRAWS), len(DRAWS[0])
    images = rng.randint(0, 256, (B, N, 45, 80, 3)).astype(np.uint8)
    fH, fW = FINAL
    out = np.zeros((B, N, 3, fH, fW), np.float32)
    packed = np.zeros((B, N, 7), np.float64)
    for b in range(B):
        for n, (resize, dims, (x0, y0), flip, rotate) in enumerate(DRAWS[b]):
            im = Image.fromarray(images[b, n]).resize(dims).crop((x0, y0, x0 + fW, y0 + fH))
            if flip:
                im = im.transpose(Image.FLIP_LEFT_RIGHT)
            out[b, n] = TF.normalize(TF.to_tensor(im.rotate(rotate)), MEAN, STD).numpy()
            packed[b, n] = [resize, dims[0], dims[1], x0, y0, float(flip), rotate]
    np.savez_compressed(OUT, images=images, draws=packed, final_dim=np.array(FINAL), mean=np.array(MEAN),
                        std=np.array(STD), out=out, pillow_version=np.array(PIL.__version__))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
