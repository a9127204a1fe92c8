"""Golden fixture for the reference's ``inputRes`` (ops.resize_u8, davis.to_device(input_res=...)), produced by the
UNMODIFIED reference dataset and transforms.

Run in the build container only (needs /root/reference, cv2 and Pillow; none is needed to USE the fixture):

    python tests/golden/make_golden_resize.py

It rebuilds the DAVIS-layout tree of ``reference_davis.npz`` from its ``file:`` entries (the same JPEG and PNG bytes),
then imports the reference's own ``dataloaders`` package with a ``scipy.misc`` stub whose ``imresize`` restates scipy
1.0's uint8 path: ``bytescale`` leaves uint8 input as it is, ``toimage`` makes an ``RGB`` image of [H,W,3] and an ``L``
image of [H,W], and the size argument is (h, w), an int percentage or a float fraction; the result is
``Image.resize((w, h), BILINEAR or NEAREST)``.  Stored in ``reference_resize.npz``:
  - ``res.<r>``: the inputRes values (``res.<r>.kind`` = tuple / int / float);
  - ``pair.<r>.<rel image path>.image`` / ``.gt``: make_img_gt_pair with inputRes = res.<r> of every frame of the
    train and val splits and of sequence ``aa`` in test mode (its unannotated frames keep a stored-size gt there);
  - ``aug.<k>.*``: RandomHorizontalFlip + ScaleNRotate of seeded train items at ``aug.<k>.res``, draws replayed as
    make_golden_davis.py does.
"""
import os
import random
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import davis_fixture                                   # noqa: E402
from make_golden_davis import AUG_SEEDS, REF          # noqa: E402

# downscale, upscale, non-uniform (height down, width up), an int percentage, a float fraction
RESOLUTIONS = [(24, 32), (64, 96), (20, 90), 60, 0.75]
AUG_RES = [(24, 32), (64, 96), 60, 0.75, (20, 90), (24, 32)]


def imresize(arr, size, interp="bilinear", mode=None):
    """scipy 1.0's scipy.misc.imresize for uint8 input."""
    from PIL import Image
    arr = np.asarray(arr)
    assert arr.dtype == np.uint8 and mode is None and arr.ndim in (2, 3)
    im = Image.fromarray(arr)
    if np.issubdtype(type(size), np.signedinteger):
        size = tuple((np.array(im.size) * (size / 100.0)).astype(int))
    elif np.issubdtype(type(size), np.floating):
        size = tuple((np.array(im.size) * size).astype(int))
    else:
        size = (size[1], size[0])
    resample = {"nearest": 0, "lanczos": 1, "bilinear": 2, "bicubic": 3, "cubic": 3}[interp]
    return np.array(im.resize(tuple(int(v) for v in size), resample=resample))


def import_reference():
    misc = types.ModuleType("scipy.misc")
    misc.imresize = imresize
    sys.modules["scipy.misc"] = misc
    sys.path.insert(0, REF)
    from dataloaders import custom_transforms as tr
    from dataloaders import davis_2016 as db
    return db, tr


def _res_entry(fx, key, res):
    fx[key] = np.array(res)
    fx[key + ".kind"] = np.array("tuple" if isinstance(res, tuple) else type(res).__name__)


def main():
    import PIL
    db, tr = import_reference()
    fx = {"pillow_version": np.array(PIL.__version__)}
    root = tempfile.mkdtemp()
    try:
        davis_fixture.write_tree(davis_fixture.load(), root)
        for r, res in enumerate(RESOLUTIONS):
            _res_entry(fx, f"res.{r}", res)
            for kw in (dict(train=True), dict(train=False), dict(train=False, seq_name="aa")):
                d = db.DAVIS2016(db_root_dir=root, inputRes=res, **kw)
                for i in range(len(d)):
                    img, gt = d.make_img_gt_pair(i)
                    key = d.img_list[i] + ("" if d.labels[i] is not None else ":nolabel")
                    fx[f"pair.{r}.{key}.image"] = img
                    fx[f"pair.{r}.{key}.gt"] = np.asarray(gt, dtype=np.float32)
        fx["res.n"] = np.array(len(RESOLUTIONS))
        for k, (seed, res) in enumerate(zip(AUG_SEEDS, AUG_RES)):
            d = db.DAVIS2016(db_root_dir=root, train=True, inputRes=res)
            idx = k % len(d)
            random.seed(seed)
            sample = d[idx]
            sample["gt"] = sample["gt"].astype(np.float32)      # as make_golden_davis.py (numpy 2 casting)
            sample = tr.RandomHorizontalFlip()(sample)
            sample = tr.ScaleNRotate(rots=(-30, 30), scales=(.75, 1.25))(sample)
            random.seed(seed)
            flip = random.random() < 0.5
            rot = (30 - -30) * random.random() - (30 - -30) / 2
            sc = (1.25 - .75) * random.random() - (1.25 - .75) / 2 + 1
            _res_entry(fx, f"aug.{k}.res", res)
            fx[f"aug.{k}.index"] = np.array(idx)
            fx[f"aug.{k}.draws"] = np.array([float(flip), rot, sc], dtype=np.float64)
            fx[f"aug.{k}.image"] = sample["image"].astype(np.float32)
            fx[f"aug.{k}.gt"] = sample["gt"].astype(np.float32)
            print(f"aug {k}: {d.img_list[idx]} res={res} flip={flip} rot={rot:.3f} sc={sc:.4f} "
                  f"shape={sample['image'].shape}")
        fx["aug.n"] = np.array(len(AUG_SEEDS))
    finally:
        shutil.rmtree(root)
    path = os.path.join(HERE, "reference_resize.npz")
    np.savez_compressed(path, **fx)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
