"""A/B of programmatic dependent launch (OSVOS_PDL=0 vs 1) on the two graphed hot loops - development aid.
(The engine switches PDL on for the inference pass whatever OSVOS_PDL says (osvos_set_pdl), so the inference arms should
match; OSVOS_PDL decides the training graph.)

    python scripts/pdl_ab.py [out_dir]

Each arm runs in its own process (the library reads OSVOS_PDL once): 480x854 inference replayed from the engine's
CUDA graph and the fwd+loss+bwd micro-batch graph (training.GraphedTrainStep).  The parent compares the arms'
outputs (inference logits must be bit-identical; gradients agree up to atomic-order noise) and prints both timings.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def worker(out_path):
    import torch
    from oracle import osvos_oracle as oc
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS, he_init_
    from osvos_pytorch_b200.training import GraphedTrainStep
    dev = torch.device("cuda", 0)
    res = {"pdl": os.environ.get("OSVOS_PDL", "0")}
    net = he_init_(OSVOS(pretrained=0, verbose=False), seed=0).to(dev).eval()
    frames = [oc.synthetic_frame(1, 480, 854, 1234 + i) for i in range(4)]
    xs = [f[0].to(dev) for f in frames]
    gts = [f[1].to(dev) for f in frames]

    def timed(fn, k):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(k):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / k

    with torch.no_grad():
        for i in range(20):
            net(xs[i % 4])
        res["infer_ms"] = min(timed(lambda i: net(xs[i % 4]), 300) for _ in range(3))
        outs = [o.clone() for o in net(xs[0])]
    res["infer_fps"] = 1000.0 / res["infer_ms"]
    for prec_h, prec_w in ((240, 427),):
        x2, _ = oc.synthetic_frame(1, prec_h, prec_w, 7)
        with torch.no_grad():
            for _ in range(5):
                net(x2.to(dev))
            res["infer240_ms"] = min(timed(lambda i: net(x2.to(dev, non_blocking=True)), 200) for _ in range(2))

    net.train()
    sample = {"image": xs[0], "gt": gts[0]}
    gstep = GraphedTrainStep(net, lambda o, gt: cbce(o[-1], gt, size_average=False), sample)
    for i in range(5):
        gstep({"image": xs[i % 4], "gt": gts[i % 4]})
    res["train_ms"] = min(timed(lambda i: gstep({"image": xs[i % 4], "gt": gts[i % 4]}), 60) for _ in range(3))
    res["train_fps"] = 1000.0 / res["train_ms"]
    net.zero_grad(set_to_none=False)
    loss = gstep(sample)
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().cpu().clone() for n, p in net.named_parameters() if p.grad is not None}
    torch.save({"outs": [o.cpu() for o in outs], "grads": grads, "loss": float(loss), "res": res}, out_path)
    print(json.dumps(res))


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "results")
    os.makedirs(out_dir, exist_ok=True)
    import torch
    arms = {}
    for pdl in ("0", "1"):
        path = os.path.join(out_dir, f"pdl_ab_{pdl}.pt")
        env = dict(os.environ, OSVOS_PDL=pdl)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", path], env=env, timeout=600)
        if r.returncode != 0:
            print(f"arm OSVOS_PDL={pdl} FAILED with exit code {r.returncode}")
            return 1
        arms[pdl] = torch.load(path)
        os.remove(path)
    a, b = arms["0"], arms["1"]
    same = all(torch.equal(x, y) for x, y in zip(a["outs"], b["outs"]))
    worst = max(float((a["grads"][n] - b["grads"][n]).norm() / (a["grads"][n].norm() + 1e-30)) for n in a["grads"])
    print(f"inference outputs bit-identical across arms: {same}")
    print(f"worst per-parameter relative gradient difference across arms: {worst:.2e} (atomic-order noise expected ~1e-6); "
          f"loss {a['loss']:.4f} vs {b['loss']:.4f}")
    for k in ("infer_ms", "infer240_ms", "train_ms"):
        print(f"{k:12s} PDL off {a['res'][k]:.4f}  on {b['res'][k]:.4f}  ratio {a['res'][k] / b['res'][k]:.4f}")
    return 0 if same and worst < 1e-3 else 2


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--worker":
        worker(sys.argv[2])
    else:
        sys.exit(main())
