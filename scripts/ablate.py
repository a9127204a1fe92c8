"""Timing ablations of the wgmma conv kernel (OSVOS_ABLATE bit mask, csrc/conv_common.cuh) - development aid.

    python scripts/ablate.py [H W] [masks...]

For each mask a fresh process (the library reads the variable once) times every conv3x3 launch of one forward with
CUDA events (best of 7 eager passes).  Results under an ablation are garbage; only the durations mean something:
1 = no weight TMA loads, 2 = no activation TMA loads, 4 = no wgmma, 8 = no epilogue stores, 16 = no epilogue at all.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def worker(h, w):
    import torch
    torch.set_grad_enabled(False)
    from oracle import osvos_oracle as oc
    import osvos_pytorch_b200.ops as O
    import osvos_pytorch_b200.engine as eng
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS, he_init_
    net = he_init_(OSVOS(pretrained=0, verbose=False)).cuda().eval()
    net._engine.use_cuda_graph = False
    x, _ = oc.synthetic_frame(1, h, w, 1234)
    x = x.cuda()
    rec = []
    orig = {}

    def wrap(name):
        f = getattr(O, name)
        orig[name] = f

        def g(*a, **k):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            r = f(*a, **k)
            e.record()
            d = name
            if name == "conv3x3":
                d += " " + "x".join(str(v) for v in a[0].shape[1:]) + f"->{a[3]}"
            rec.append((d, s, e))
            return r
        setattr(O, name, g)
        setattr(eng.ops, name, g)
    for n in ("conv_first", "conv3x3", "tail_fwd"):
        wrap(n)
    best = None
    for rep in range(8):
        rec.clear()
        net(x)
        torch.cuda.synchronize()
        t = [(d, s.elapsed_time(e) * 1e3) for d, s, e in rec]
        if rep == 0:
            continue
        best = t if best is None else [(d, min(a, b)) for (d, a), (_, b) in zip(best, t)]
    print("RESULT " + json.dumps(best))


def main():
    args = sys.argv[1:]
    h, w = (int(args[0]), int(args[1])) if len(args) >= 2 else (480, 854)
    masks = [int(v) for v in args[2:]] or [0, 1, 2, 3, 4, 8, 12, 7, 15, 16]
    table = {}
    for m in masks:
        env = dict(os.environ, OSVOS_ABLATE=str(m))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", str(h), str(w)], env=env,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
        line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
        if not line:
            print(f"mask {m}: FAILED\n{r.stdout[-2000:]}")
            continue
        table[m] = json.loads(line[0][7:])
    names = [d for d, _ in table[masks[0]]]
    print(f"# {h}x{w} exact, per-launch CUDA-event us (best of 7); columns = OSVOS_ABLATE mask "
          "(1 no weight loads, 2 no activation loads, 4 no MMAs, 8 no epilogue stores, 16 no epilogue)")
    print(f"{'launch':34s}" + "".join(f"{m:>9d}" for m in table))
    for i, d in enumerate(names):
        print(f"{d:34s}" + "".join(f"{table[m][i][1]:9.1f}" for m in table))
    print(f"{'sum':34s}" + "".join(f"{sum(v for _, v in table[m]):9.1f}" for m in table))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--worker":
        worker(int(sys.argv[2]), int(sys.argv[3]))
    else:
        main()
