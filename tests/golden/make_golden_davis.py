"""Golden fixture for the native DAVIS-2016 loader (osvos_pytorch_b200.davis and csrc/frames.cu), produced by the
UNMODIFIED reference dataset and transforms.

Run in the build container only (needs /root/reference and cv2; neither is needed to USE the fixture):

    python tests/golden/make_golden_davis.py

It writes a small DAVIS-layout tree (JPEG frames, 0/255 PNG masks plus one all-zero and one non-binary mask, three
sequences at odd sizes), then imports the reference's own ``dataloaders`` package (davis_2016.py, helpers.py,
custom_transforms.py, no edits) with a ``scipy.misc`` stub: ``imresize`` is gone from SciPy and the import alone would
fail; the stub raises if it is ever called.  Stored in ``reference_davis.npz``:
  - ``file:<path>``: the encoded bytes of every file of the tree, so tests rebuild the identical tree without encoding;
  - ``list.<mode>.img`` / ``.labels`` (``""`` for None) / ``.fname``: the dataset's lists for the train split, the val
    split and sequence mode (train=True and train=False);
  - ``pair.<rel image path>.image`` / ``.gt``: make_img_gt_pair of every frame of the splits and of the sequences;
  - ``aug.<k>.*``: the reference's RandomHorizontalFlip + ScaleNRotate on seeded items of the train split (mask as
    float32, see main), with the draws replayed in the transforms' order.
"""
import os
import random
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"

# sequence -> (height, width, frames)
SEQS = {"aa": (33, 45, 3), "bb": (48, 70, 2), "cc": (97, 131, 2)}
TRAIN, VAL = ["aa", "cc"], ["bb"]
AUG_SEEDS = [200, 201, 202, 203, 204, 205]


def _mask(rng, h, w, seq, i):
    yy, xx = np.mgrid[0:h, 0:w]
    blob = ((yy - h * (0.4 + 0.05 * i)) ** 2 / (h * 0.3) ** 2 + (xx - w * 0.55) ** 2 / (w * 0.25) ** 2) < 1.0
    m = (blob ^ (rng.random((h, w)) > 0.97)).astype(np.uint8) * 255
    if (seq, i) == ("bb", 1):
        m[:] = 0                                         # an annotated frame with no object
    if (seq, i) == ("cc", 0):
        m = np.where(m > 0, 255, np.where(rng.random((h, w)) > 0.9, 128, 0)).astype(np.uint8)   # non-binary
    return m


def write_tree(root, cv2):
    rng = np.random.default_rng(77)
    for seq, (h, w, frames) in SEQS.items():
        os.makedirs(os.path.join(root, "JPEGImages/480p", seq))
        os.makedirs(os.path.join(root, "Annotations/480p", seq))
        yy, xx = np.mgrid[0:h, 0:w]
        for i in range(frames):
            base = np.stack([(xx * 255 // w), (yy * 255 // h), ((xx + yy + 40 * i) * 3) % 256], -1)
            img = np.clip(base + rng.integers(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(root, "JPEGImages/480p", seq, "%05d.jpg" % i), img)
            cv2.imwrite(os.path.join(root, "Annotations/480p", seq, "%05d.png" % i), _mask(rng, h, w, seq, i))
    with open(os.path.join(root, "train_seqs.txt"), "w") as f:
        f.write("".join(s + "\n" for s in TRAIN))
    with open(os.path.join(root, "val_seqs.txt"), "w") as f:
        f.write("".join(s + "\n" for s in VAL))


def import_reference():
    misc = types.ModuleType("scipy.misc")

    def imresize(*args, **kwargs):
        raise AssertionError("scipy.misc.imresize called: the fixture never sets inputRes")
    misc.imresize = imresize
    sys.modules["scipy.misc"] = misc
    sys.path.insert(0, REF)
    from dataloaders import custom_transforms as tr
    from dataloaders import davis_2016 as db
    return db, tr


def main():
    import cv2
    db, tr = import_reference()
    fx = {"cv2_version": np.array(cv2.__version__)}
    root = tempfile.mkdtemp()
    try:
        write_tree(root, cv2)
        for dirpath, _, files in os.walk(root):
            for f in files:
                rel = os.path.relpath(os.path.join(dirpath, f), root)
                fx["file:" + rel] = np.fromfile(os.path.join(dirpath, f), dtype=np.uint8)
        modes = {"train": dict(train=True), "val": dict(train=False),
                 "seq_train": dict(train=True, seq_name="aa"), "seq_test": dict(train=False, seq_name="aa")}
        for mode, kw in modes.items():
            d = db.DAVIS2016(db_root_dir=root, **kw)
            fx[f"list.{mode}.img"] = np.array(d.img_list)
            fx[f"list.{mode}.labels"] = np.array(["" if v is None else v for v in d.labels])
            fx[f"list.{mode}.fname"] = np.array([d[i].get("fname", "") for i in range(len(d))])
            for i in range(len(d)):
                img, gt = d.make_img_gt_pair(i)
                key = d.img_list[i] + ("" if d.labels[i] is not None else ":nolabel")
                fx[f"pair.{key}.image"] = img
                fx[f"pair.{key}.gt"] = gt
        d = db.DAVIS2016(db_root_dir=root, train=True)
        for k, seed in enumerate(AUG_SEEDS):
            idx = k % len(d)
            random.seed(seed)
            sample = d[idx]
            # numpy >= 2 makes gt / np.max([gt.max(), 1e-8]) float64; numpy 1 (value-based casting, the reference's
            # era) kept it float32.  The values are the same, but OpenCV 4.13's INTER_NEAREST warpAffine of a float64
            # array does not follow its fixed-point algorithm (the float32 path does: reference_augment.npz), so the
            # transforms get the float32 mask the reference was written against.
            sample["gt"] = sample["gt"].astype(np.float32)
            sample = tr.RandomHorizontalFlip()(sample)
            sample = tr.ScaleNRotate(rots=(-30, 30), scales=(.75, 1.25))(sample)
            random.seed(seed)                       # replay the draws in the transforms' order (:92, :25-29)
            flip = random.random() < 0.5
            rot = (30 - -30) * random.random() - (30 - -30) / 2
            sc = (1.25 - .75) * random.random() - (1.25 - .75) / 2 + 1
            fx[f"aug.{k}.index"] = np.array(idx)
            fx[f"aug.{k}.draws"] = np.array([float(flip), rot, sc], dtype=np.float64)
            fx[f"aug.{k}.image"] = sample["image"].astype(np.float32)
            fx[f"aug.{k}.gt"] = sample["gt"].astype(np.float32)
            print(f"aug {k}: {d.img_list[idx]} flip={flip} rot={rot:.3f} sc={sc:.4f}")
        fx["aug.n"] = np.array(len(AUG_SEEDS))
    finally:
        shutil.rmtree(root)
    path = os.path.join(HERE, "reference_davis.npz")
    np.savez_compressed(path, **fx)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
