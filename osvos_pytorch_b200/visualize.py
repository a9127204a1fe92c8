"""Overlays of a results folder (DESIGN.md §25): each result PNG drawn over its DAVIS frame on the GPU and written as
a JPEG file and / or one MJPEG video per sequence.

``render_results`` chains decode -> draw -> encode over a folder the way evaluation.score_results chains decode ->
score: reader threads read and parse the files while the device decodes (jpeg.decode_files, png.decode_files), draws
(ops.overlay_labels) and encodes (ops.encode_jpeg) the previous batch."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import jpeg, ops, png
from . import video as _video

RED = b"\0\0\0\xff\0\0"                  # entry 1 = RGB red: BGR (0, 0, 255), overlay_mask's default colour


def _stems(folder, ext):
    return sorted(f[:-len(ext)] for f in os.listdir(folder) if f.lower().endswith(ext))


def render_results(results_dir, db_root_dir=None, sequences=None, davis="2016", threshold=128, quality=95,
                   frames=True, video=False, fps=24.0, out_dir=None, device="cuda", batch=16, decode="device",
                   readers=4, palette=None):
    """Draws every result of ``results_dir`` over its frame and writes ``out_dir/<seq>_overlay/<stem>.jpg``
    (``frames``) and / or ``out_dir/<seq>_overlay.avi`` (``video``, MJPEG at ``fps`` whose frames are those JPEG
    files byte for byte).  ``out_dir`` defaults to ``results_dir``.

    ``results_dir/<seq>/<stem>.png`` is drawn over ``db_root_dir/JPEGImages/480p/<seq>/<stem>.jpg``; a result without
    a frame raises ValueError, annotations are not read.  ``sequences``: default those of ``val_seqs.txt`` (2016) or
    ``ImageSets/2017/val.txt`` (2017) that have a folder under ``results_dir``.

    ``davis="2016"``: the object is ``byte >= threshold`` (128 is logit > 0 for "mask" and "prob" files), drawn in
    red: for mask files the JPEGs equal train_online.py --overlay's.  ``davis="2017"``: the results are decoded to
    their indices (palette files) and each id is drawn in the colour of the file's own PLTE, else of the DAVIS
    palette; ``palette`` (PLTE bytes) overrides both.  Results at another size than their frame are resized to it
    first (ops.resize_u8, nearest, which keeps ids).  Each overlay is encoded with ops.encode_jpeg(``quality``): the
    bytes cv2.imencode writes for the drawn frame.

    ``decode``: "device" parses the files in ``readers`` threads and decodes them on the GPU (cv2 / Pillow for files
    outside the decoders' subsets or flagged by them); "host" decodes every file with cv2 / Pillow.  The written files
    are the same either way.  A batch never mixes sequences.  Returns {'sequences': {seq: frames drawn}, 'frames',
    'fallback_files', 'redecoded_files'}."""
    if decode not in ("device", "host"):
        raise ValueError(f"decode must be 'device' or 'host', got {decode!r}")
    if davis not in ("2016", "2017"):
        raise ValueError(f"davis must be '2016' or '2017', got {davis!r}")
    if not 1 <= int(quality) <= 100:
        raise ValueError(f"quality must lie in 1..100, got {quality}")
    if not frames and not video:
        raise ValueError("nothing to write: ask for frames, a video or both")
    if fps <= 0:
        raise ValueError(f"fps must be positive, got {fps}")
    multi = davis == "2017"
    if palette is not None and not multi:
        raise ValueError("palette applies to davis='2017' label maps; DAVIS-2016 results are drawn in red")
    if db_root_dir is None:
        from mypath import Path
        db_root_dir = Path.db_root_dir()
    out_dir = results_dir if out_dir is None else out_dir
    img_root = os.path.join(db_root_dir, "JPEGImages", "480p")
    if sequences is None:
        listing = os.path.join("ImageSets", "2017", "val.txt") if multi else "val_seqs.txt"
        with open(os.path.join(db_root_dir, listing)) as f:
            sequences = [s.strip() for s in f if s.strip()]
        sequences = [s for s in sequences if os.path.isdir(os.path.join(results_dir, s))]
        if not sequences:
            raise ValueError(f"no sequence of {listing} has a folder under {results_dir}")
    pairs = []                                               # (sequence, stem, result path, frame path)
    for seq in sequences:
        res_dir, img_dir = os.path.join(results_dir, seq), os.path.join(img_root, seq)
        if not os.path.isdir(res_dir) or not os.path.isdir(img_dir):
            raise ValueError(f"unknown sequence {seq!r}: no folder " + (res_dir if not os.path.isdir(res_dir) else img_dir))
        have = set(_stems(img_dir, ".jpg"))
        stems = _stems(res_dir, ".png")
        missing = [s for s in stems if s not in have]
        if missing:
            raise ValueError(f"sequence {seq!r}: no frame for result(s) {', '.join(missing[:5])} in {img_dir}")
        pairs.extend((seq, s, os.path.join(res_dir, s + ".png"), os.path.join(img_dir, s + ".jpg")) for s in stems)
    mode = "index" if multi else None
    fixed = None if palette is None else bytes(palette)

    def read(pair):
        with open(pair[2], "rb") as f:
            res = f.read()
        with open(pair[3], "rb") as f:
            img = f.read()
        pal = (fixed or png.palette_of(res) or png.davis_palette()) if multi else RED
        if decode == "device":
            return (res, png.parse(res, palette=mode)), (img, jpeg.parse(img)), pal
        return ((png.decode_host_index(res) if multi else png.decode_host(res)), None), (jpeg.decode_host(img), None), pal

    def to_device(items, decoder):
        if decode == "device":
            return decoder([d for d, _ in items], device, parsed=[p for _, p in items])
        if len({m.shape for m, _ in items}) != 1:
            raise ValueError("the files differ in size")
        return torch.from_numpy(np.stack([m for m, _ in items])).to(device), 0, 0

    def decode_results(datas, dev, parsed):
        return png.decode_files(datas, dev, parsed=parsed, palette=mode)

    drawn, fallback, redecoded = {}, 0, 0
    threshold = int(threshold)
    with ThreadPoolExecutor(max(1, int(readers))) as pool:
        loaded = pool.map(read, pairs)
        start = 0
        while start < len(pairs):
            seq = pairs[start][0]
            stop = start
            while stop < len(pairs) and stop - start < batch and pairs[stop][0] == seq:
                stop += 1
            items = [next(loaded) for _ in range(stop - start)]
            try:
                res, fb_r, rd_r = to_device([it[0] for it in items], decode_results)
                img, fb_i, rd_i = to_device([it[1] for it in items], jpeg.decode_files)
            except ValueError as e:
                raise ValueError(f"sequence {seq!r}, results {pairs[start][1]} .. {pairs[stop - 1][1]}: {e}") from e
            fallback += fb_r + fb_i
            redecoded += rd_r + rd_i
            labels = res if multi else (res >= threshold).to(torch.uint8)
            h, w = int(img.shape[1]), int(img.shape[2])
            if tuple(labels.shape[1:]) != (h, w):
                labels = ops.resize_u8(labels, (h, w), mode="nearest")
            a = 0                                            # one call per run of results sharing a palette
            while a < len(items):
                b = a + 1
                while b < len(items) and items[b][2] == items[a][2]:
                    b += 1
                ops.overlay_labels(img[a:b], labels[a:b], items[a][2], out=img[a:b])
                a = b
            enc, lengths = ops.encode_jpeg(img, quality)
            lengths = lengths.cpu().tolist()                 # one wait per batch
            host = enc[:, :max(lengths)].cpu().numpy()
            files = [host[i, :lengths[i]].tobytes() for i in range(len(items))]
            if seq not in drawn:
                drawn[seq], clip = 0, []
                if frames:
                    os.makedirs(os.path.join(out_dir, seq + "_overlay"), exist_ok=True)
            if frames:
                for (_, stem, _, _), data in zip(pairs[start:stop], files):
                    with open(os.path.join(out_dir, seq + "_overlay", stem + ".jpg"), "wb") as f:
                        f.write(data)
            drawn[seq] += len(files)
            if video:
                clip += files
                if stop == len(pairs) or pairs[stop][0] != seq:
                    os.makedirs(out_dir, exist_ok=True)
                    _video.write_avi(os.path.join(out_dir, seq + "_overlay.avi"), clip, fps)
            start = stop
    return {"sequences": drawn, "frames": len(pairs),
            "fallback_files": fallback, "redecoded_files": redecoded}
