"""Device JPEG decode time per 480x854 frame (CUDA events, ops.decode_jpeg) at batch 1 and 12, quality 75 and 95,
against single-thread cv2.imdecode on the same host, in alternated rounds, with the host's jpeg.parse + jpeg.pack time
per frame (what a DataLoader worker does instead of decoding); then DeviceFrames build time for a 240-frame tree at
1 / 2 / 4 workers, host decode against device decode.  Prints the GPU's name and power limit.  Frames are made as
scripts/time_data.py makes them; the tree goes to a temporary directory.  Prints one JSON line."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def frame(seed, h=480, w=854):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:h, :w]
    base = np.stack([x * 255 // (w - 1), y * 255 // (h - 1), ((x // 40 + y // 40) % 2) * 200], -1)
    return np.clip(base + rng.integers(-20, 20, (h, w, 3)), 0, 255).astype(np.uint8)


def _store_builds(cv2, seqs=8, per_seq=30):
    """DeviceFrames build seconds for a seqs x per_seq frame train split (q75 frames, binary masks), alternating host
    and device decode at 1, 2 and 4 workers; the stores are checked equal."""
    import tempfile
    from osvos_pytorch_b200 import davis
    out = {}
    with tempfile.TemporaryDirectory() as root:
        with open(os.path.join(root, "train_seqs.txt"), "w") as f:
            f.write("\n".join(f"s{k}" for k in range(seqs)) + "\n")
        for k in range(seqs):
            for sub in ("JPEGImages", "Annotations"):
                os.makedirs(os.path.join(root, sub, "480p", f"s{k}"))
            for i in range(per_seq):
                img = frame(1000 * k + i)
                cv2.imwrite(os.path.join(root, "JPEGImages", "480p", f"s{k}", f"{i:05d}.jpg"), img,
                            [cv2.IMWRITE_JPEG_QUALITY, 75])
                cv2.imwrite(os.path.join(root, "Annotations", "480p", f"s{k}", f"{i:05d}.png"),
                            ((img[..., 1] > 128) * 255).astype(np.uint8))
        for workers in (1, 2, 4):
            for decode in ("host", "device", "host", "device"):
                st = davis.DeviceFrames(davis.DAVIS2016Frames(db_root_dir=root, decode=decode), "cuda", workers=workers)
                out.setdefault(f"{decode}_w{workers}", []).append(round(st.build_s, 2))
                if decode == "host":
                    ref = st.groups[0]["img"]
                else:
                    assert torch.equal(ref, st.groups[0]["img"])
                del st
    return out


def main():
    import cv2
    from osvos_pytorch_b200 import jpeg, ops
    cv2.setNumThreads(1)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    res = {"gpu": gpu}
    rounds = 5
    for q in (75, 95):
        bufs = [cv2.imencode(".jpg", frame(s), [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes() for s in range(12)]
        res[f"q{q}_kb"] = round(sum(map(len, bufs)) / len(bufs) / 1024, 1)
        for b in (1, 12):
            blob = jpeg.pack([jpeg.parse(x) for x in bufs[:b]])
            dev = torch.from_numpy(blob).cuda()
            nseg = jpeg.segment_count(blob)
            out = torch.empty((b, 480, 854, 3), dtype=torch.uint8, device="cuda")
            for _ in range(3):
                ops.decode_jpeg(dev, b, 480, 854, out=out, nseg=nseg)
            dev_ms, cpu_ms, parse_ms = [], [], []
            for _ in range(rounds):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(20):
                    ops.decode_jpeg(dev, b, 480, 854, out=out, nseg=nseg)
                e1.record()
                torch.cuda.synchronize()
                dev_ms.append(e0.elapsed_time(e1) / 20 / b)
                t = time.perf_counter()
                for x in bufs[:b]:
                    cv2.imdecode(np.frombuffer(x, np.uint8), cv2.IMREAD_COLOR)
                cpu_ms.append((time.perf_counter() - t) * 1e3 / b)
                t = time.perf_counter()
                jpeg.pack([jpeg.parse(x) for x in bufs[:b]])
                parse_ms.append((time.perf_counter() - t) * 1e3 / b)
            ok = all(np.array_equal(out[i].cpu().numpy(), cv2.imdecode(np.frombuffer(bufs[i], np.uint8), 1))
                     for i in range(b))
            res[f"q{q}_b{b}"] = {"device_us_per_frame": round(1e3 * float(np.median(dev_ms)), 1),
                                 "cv2_us_per_frame": round(1e3 * float(np.median(cpu_ms)), 1),
                                 "parse_pack_us_per_frame": round(1e3 * float(np.median(parse_ms)), 1), "bit_identical": ok}
    res["device_frames_build_s"] = _store_builds(cv2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
