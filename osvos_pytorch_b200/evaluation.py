"""DAVIS-2016 region (J) and boundary (F) scores from the device counts of ``ops.davis_measures`` (DESIGN.md §14).

The kernel produces six integers per frame; this module turns them into J and F (on the device, no synchronisation)
and a sequence's per-frame series into the benchmark's statistics: mean M, recall O and decay D.  As the DAVIS-2016
benchmark does, the statistics leave out a sequence's first frame (its annotation is the network's input) and its
last frame; the per-frame values of every frame are kept, so other conventions can be recomputed from them.
"""
import math

import numpy as np
import torch

BOUND_TH = 0.008                      # boundary tolerance as a fraction of the frame diagonal


def bound_pix(h, w):
    """Boundary tolerance radius in pixels: ceil(0.008 * sqrt(h² + w²)) (8 at 480x854, 18 at 1080x1920)."""
    return int(math.ceil(BOUND_TH * math.sqrt(h * h + w * w)))


def j_and_f(counts):
    """int [N,6] counts -> (J, F), float64 [N] each, on the counts' device.  J = |P∧G| / |P∨G| (1 when both masks are
    empty); F = 2PR / (P + R) of boundary precision P and recall R, with the benchmark's rules for empty boundaries."""
    c = counts.to(torch.float64)
    inter, union, n_fg, n_gt, fg_match, gt_match = c.unbind(-1)
    one, zero = torch.ones_like(inter), torch.zeros_like(inter)
    j = torch.where(union > 0, inter / union.clamp(min=1), one)
    # both boundaries empty: P = R = 1; only B(P) empty: P = 1, R = 0; only B(G) empty: P = 0, R = 1
    prec = torch.where(n_fg > 0, torch.where(n_gt > 0, fg_match / n_fg.clamp(min=1), zero), one)
    rec = torch.where(n_gt > 0, torch.where(n_fg > 0, gt_match / n_gt.clamp(min=1), zero), one)
    s = prec + rec
    f = torch.where(s > 0, 2 * prec * rec / torch.where(s > 0, s, one), zero)
    return j, f


def decay_bins(n):
    """The first indices of the benchmark's four decay bins of an n-frame series, plus the last index."""
    return (np.round(np.linspace(1, n, 5) + 1e-10) - 1).astype(int)


def statistics(values):
    """A sequence's per-frame series (every frame, first and last included) -> {'M', 'O', 'D'} over frames 1 .. n-2:
    M = mean, O = fraction above 0.5, D = mean of the first quarter bin minus mean of the last.  NaN when no frame
    is left."""
    x = np.asarray(values.cpu() if torch.is_tensor(values) else values, dtype=np.float64)[1:-1]
    if x.size == 0:
        return {"M": float("nan"), "O": float("nan"), "D": float("nan")}
    i = decay_bins(x.size)
    return {"M": float(np.mean(x)), "O": float(np.mean(x > 0.5)),
            "D": float(np.mean(x[i[0]:i[1] + 1]) - np.mean(x[i[3]:i[4] + 1]))}


class SequenceScores:
    """Accumulates device counts frame by frame without synchronising; ``result()`` reads them back once."""

    def __init__(self):
        self._counts = []

    def add(self, counts):
        self._counts.append(counts.reshape(-1, 6))

    def result(self):
        """{'J': per-frame list, 'F': per-frame list, 'counts': per-frame lists of six ints,
        'statistics': {'J': {M, O, D}, 'F': {M, O, D}}}."""
        if not self._counts:
            counts = torch.zeros((0, 6), dtype=torch.int32)
        else:
            counts = torch.cat([c.to(self._counts[0].device) for c in self._counts]).cpu()
        j, f = j_and_f(counts)
        return {"J": j.tolist(), "F": f.tolist(), "counts": counts.tolist(),
                "statistics": {"J": statistics(j), "F": statistics(f)}}


def dataset_scores(per_seq):
    """{sequence: SequenceScores or its result()} -> the dataset figures {'J': {M, O, D}, 'F': {M, O, D}}: the mean over
    sequences of the per-sequence statistics (NaN without sequences)."""
    stats = [(sc.result() if isinstance(sc, SequenceScores) else sc)["statistics"] for sc in per_seq.values()]
    return {m: {k: float(np.mean([st[m][k] for st in stats])) if stats else float("nan") for k in "MOD"}
            for m in ("J", "F")}


def _png_stems(folder):
    import os
    return sorted(f[:-4] for f in os.listdir(folder) if f.lower().endswith(".png"))


def score_results(results_dir, db_root_dir=None, sequences=None, threshold=128, device="cuda", batch=16,
                  decode="device", readers=4):
    """Scores a folder of result PNGs against the DAVIS-2016 annotations (DESIGN.md §22).

    ``results_dir/<seq>/<stem>.png`` is paired with ``db_root_dir/Annotations/480p/<seq>/<stem>.png`` by file stem;
    a missing result, a missing annotation or differing sizes raise ValueError.  ``sequences``: the sequences to score
    (default: those of ``val_seqs.txt`` that have a folder under ``results_dir``).  The prediction is
    ``byte >= threshold`` (128 is logit > 0 for "mask" and "prob" files), the annotation ``byte != 0``, scored by
    ops.davis_measures with no per-frame synchronisation.  ``decode``: "device" reads and parses the files in
    ``readers`` threads and decodes them with png.decode_files (cv2 for files outside its subset or flagged by it),
    "host" decodes every file with cv2; both give the same counts.

    Returns {'sequences': {seq: SequenceScores.result()}, 'dataset': dataset_scores(...), 'frames', 'fallback_files',
    'redecoded_files'}."""
    import os
    from concurrent.futures import ThreadPoolExecutor

    from . import ops, png
    if decode not in ("device", "host"):
        raise ValueError(f"decode must be 'device' or 'host', got {decode!r}")
    if db_root_dir is None:
        from mypath import Path
        db_root_dir = Path.db_root_dir()
    ann_root = os.path.join(db_root_dir, "Annotations", "480p")
    if sequences is None:
        with open(os.path.join(db_root_dir, "val_seqs.txt")) as f:
            sequences = [s.strip() for s in f if s.strip()]
        sequences = [s for s in sequences if os.path.isdir(os.path.join(results_dir, s))]
        if not sequences:
            raise ValueError(f"no sequence of val_seqs.txt has a folder under {results_dir}")
    pairs = []                                               # (sequence, result path, annotation path)
    for seq in sequences:
        res_dir, ann_dir = os.path.join(results_dir, seq), os.path.join(ann_root, seq)
        if not os.path.isdir(res_dir) or not os.path.isdir(ann_dir):
            raise ValueError(f"unknown sequence {seq!r}: no folder " + (res_dir if not os.path.isdir(res_dir) else ann_dir))
        have, want = set(_png_stems(res_dir)), _png_stems(ann_dir)
        missing = [s for s in want if s not in have]
        if missing:
            raise ValueError(f"sequence {seq!r}: no result for frame(s) {', '.join(missing[:5])} in {res_dir}")
        extra = sorted(have - set(want))
        if extra:
            raise ValueError(f"sequence {seq!r}: no annotation for result(s) {', '.join(extra[:5])} in {ann_dir}")
        pairs.extend((seq, os.path.join(res_dir, s + ".png"), os.path.join(ann_dir, s + ".png")) for s in want)

    def read(path):
        with open(path, "rb") as f:
            data = f.read()
        return (data, png.parse(data)) if decode == "device" else (png.decode_host(data), None)

    def to_device(items):
        if decode == "device":
            return png.decode_files([d for d, _ in items], device, parsed=[p for _, p in items])
        if len({m.shape for m, _ in items}) != 1:
            raise ValueError("the files differ in size")
        return torch.from_numpy(np.stack([m for m, _ in items])).to(device), 0, 0

    scores = {seq: SequenceScores() for seq in sequences}
    fallback = redecoded = 0
    threshold = int(threshold)
    with ThreadPoolExecutor(max(1, int(readers))) as pool:
        loaded = pool.map(lambda pr: (read(pr[1]), read(pr[2])), pairs)
        # one batch never mixes sequences: a sequence has one size, the dataset need not
        start = 0
        while start < len(pairs):
            seq = pairs[start][0]
            stop = start
            while stop < len(pairs) and stop - start < batch and pairs[stop][0] == seq:
                stop += 1
            items = [next(loaded) for _ in range(stop - start)]
            try:
                res, fb_r, rd_r = to_device([it[0] for it in items])
                ann, fb_a, rd_a = to_device([it[1] for it in items])
            except ValueError as e:
                raise ValueError(f"sequence {seq!r}, frames {os.path.basename(pairs[start][1])} .. "
                                 f"{os.path.basename(pairs[stop - 1][1])}: {e}") from e
            if res.shape != ann.shape:
                raise ValueError(f"sequence {seq!r}: results are {res.shape[1]}x{res.shape[2]}, annotations "
                                 f"{ann.shape[1]}x{ann.shape[2]}")
            fallback += fb_r + fb_a
            redecoded += rd_r + rd_a
            pred = torch.where(res >= threshold, 1.0, -1.0).to(torch.float32)
            scores[seq].add(ops.davis_measures(pred, ann))
            start = stop
    per_seq = {seq: sc.result() for seq, sc in scores.items()}
    return {"sequences": per_seq, "dataset": dataset_scores(per_seq), "frames": len(pairs),
            "fallback_files": fallback, "redecoded_files": redecoded}
