"""Writes tests/golden/lfw_aug.npz: eight synthetic 250x250 LFW-like photos as JPEG (Pillow, quality 75, 4:2:0), their
Pillow decodes, and the rows fg_dataset_augment must build from them for seed 43 and two augmentations per photo
(tests/aug_ref.py on the descriptors fg_lfw_aug_params gives).  The GPU tests read only the npz, so the machine that
runs them needs no Pillow.  To keep the file small, the decodes and the rows are stored as SHA-256 of their planar
bytes, and four rows also keep their pixels.

    python tests/golden/make_golden_aug.py      # rewrites the npz (Pillow and the built library required)

Arrays (P photos, R = P * (1 + n_aug) rows of 3 x 64 x 64):
    names [P] str                LFW's layout, Person_Name/Person_Name_000k.jpg, in list_lfw_files order
    jpegs uint8 (all files back to back), offsets [P+1] int64
    photo_sha256 [P] str         SHA-256 (hex) of Pillow's planar [3][250][250] decode of each file
    seed, n_aug                  43, 2
    augs [R] fg_aug              fg_lfw_aug_params(seed, 0, P, n_aug, 250, 250)
    sha256 [R] str               SHA-256 of each expected row
    full_idx [4] int64, full_rows [4][3][64][64] uint8
"""
import hashlib
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from make_golden_jpeg import encode, face  # noqa: E402

import aug_ref as R  # noqa: E402

NAMES = ["Aaron_Eckhart", "Aaron_Eckhart", "Abel_Pacheco", "Ana_Guevara", "Ana_Guevara", "Ana_Guevara", "Bob_Hope",
         "Zoe_Ball"]


def photos(rng):
    out = []
    for k in range(len(NAMES)):
        img = face(rng, 250, 250)
        if k == 5:  # no dark pixels: the warp's clip has min > 0
            img = (img // 2 + 90).astype(np.uint8)
        if k == 6:  # saturated white and black blocks inside the crop box
            img[100:130, 90:120] = 255
            img[140:170, 130:160] = 0
        out.append(img)
    return out


def main():
    from PIL import Image
    from face_generator_b200.dataset import lfw_aug_params
    rng = np.random.default_rng(2026)
    names, blobs, decs = [], [], []
    counts = {}
    for name, img in zip(NAMES, photos(rng)):
        counts[name] = counts.get(name, 0) + 1
        names.append("%s/%s_%04d.jpg" % (name, name, counts[name]))
        b = encode(img, quality=75, subsampling=2)
        blobs.append(b)
        decs.append(np.asarray(Image.open(io.BytesIO(b)).convert("RGB")).transpose(2, 0, 1).copy())
    assert names == sorted(names, key=os.fsencode)
    seed, n_aug = 43, 2
    augs = lfw_aug_params(seed, 0, len(decs), n_aug, 250, 250)
    rows = R.augment_rows(np.stack(decs), augs)
    full_idx = np.array([0, 4, 17, 23], np.int64)
    offsets = np.zeros(len(blobs) + 1, np.int64)
    offsets[1:] = np.cumsum([len(b) for b in blobs])
    np.savez_compressed(
        os.path.join(HERE, "lfw_aug.npz"), names=np.array(names), jpegs=np.frombuffer(b"".join(blobs), np.uint8),
        offsets=offsets, photo_sha256=np.array([hashlib.sha256(d.tobytes()).hexdigest() for d in decs]),
        seed=np.int64(seed), n_aug=np.int64(n_aug), augs=augs,
        sha256=np.array([hashlib.sha256(r.tobytes()).hexdigest() for r in rows]), full_idx=full_idx,
        full_rows=rows[full_idx])
    print("lfw_aug.npz: %d photos, %d rows, %d JPEG bytes" % (len(decs), len(rows), offsets[-1]))


if __name__ == "__main__":
    main()
