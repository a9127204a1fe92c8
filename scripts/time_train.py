"""Per-kernel CUDA-event timing of one fwd+bwd (online objective) - development aid."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from collections import OrderedDict
from oracle import osvos_oracle as oc
import osvos_pytorch_b200.ops as O
from osvos_pytorch_b200.networks.vgg_osvos import OSVOS, he_init_
from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce

h, w = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (480, 854)
prec = sys.argv[3] if len(sys.argv) > 3 else "exact"
net = he_init_(OSVOS(pretrained=0, verbose=False, precision=prec)).cuda().train()
x, gt = oc.synthetic_frame(1, h, w, 1234)
x, gt = x.cuda(), gt.cuda()

def step():
    net.zero_grad(set_to_none=False)
    loss = cbce(net(x)[-1], gt, size_average=False)
    loss.backward()
for _ in range(3):
    step()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
reps = 10
e0.record()
for _ in range(reps):
    step()
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
print(f"fwd+bwd {h}x{w} {prec}: {ms:.3f} ms/frame = {1000/ms:.1f} fps; conv TFLOP/s (algorithmic, 3x fwd flops) {3*oc.conv_flops(h, w)/ms/1e9:.1f}")
rec = []
names = ["conv_first", "conv3x3", "maxpool2x2", "tail_fwd", "conv3x3_wgrad", "tail_bwd", "sum_f32", "side_folded_multi",
         "side_folded_wgrad_multi", "side_grads_finish", "unpool_mask", "conv_first_bwd", "pack_conv3x3_weights",
         "fold_side_weights_multi"]
def wrap(name):
    f = getattr(O, name)
    def g(*a, **k):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); r = f(*a, **k); e.record()
        d = name
        if name in ("conv3x3", "conv3x3_wgrad"):
            d += " " + "x".join(str(v) for v in a[0].shape) + f"->{a[3] if name == 'conv3x3' else a[2]}"
        rec.append((d, s, e)); return r
    setattr(O, name, g)
for nme in names:
    wrap(nme)
step(); torch.cuda.synchronize()
agg = OrderedDict()
for d, s, e in rec:
    t = s.elapsed_time(e)
    print(f"  {d:50s} {t*1000:9.1f} us")
    k = d.split(" ")[0]
    agg[k] = agg.get(k, 0) + t
print("  ---- totals")
for k, v in agg.items():
    print(f"  {k:30s} {v*1000:9.1f} us")
print(f"  sum {sum(agg.values()):.3f} ms")
