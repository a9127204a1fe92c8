"""Test-time path of the reference (train_online.py:170-189) as a device pipeline (SURVEY.md 8f item 4).

The reference loops over the sequence one frame at a time: ``img.to(device)`` -> ``net.forward`` ->
``outputs[-1].cpu()`` -> numpy sigmoid -> ``scipy.misc.imsave``; every stage waits for the previous one.
``SequenceSegmenter`` keeps the same per-frame semantics but overlaps the three legs on separate CUDA streams with
a small ring of buffers: while frame i is in the network, frame i+1 is crossing PCIe host->device and the result
of frame i-1 is crossing device->host.  The result is either the fused logit map (fp32, what ``outputs[-1]`` holds)
or the 8-bit map produced on the device by ``ops.logits_to_u8`` (``bytescale`` = the PNG payload the reference
writes, ``prob``, ``mask``), which cuts the device->host bytes by 4.
"""
import torch

from . import ops


class SequenceSegmenter:
    """``for result in SequenceSegmenter(net)(frames): ...`` - ``frames`` yields host tensors [N,3,H,W] fp32 (pinned
    for real overlap); ``result`` is a pinned host tensor [N,1,H,W] (fp32 logits or uint8) that stays valid until
    ``depth`` further frames have been consumed.  All frames of one call must share a shape.

    ``frames="bgr8"``: the frames are decoded uint8 [N,H,W,3] BGR (what cv2.imread returns) instead; only those bytes
    cross PCIe, and ops.image_from_bgr8 (float conversion and ``meanval`` subtraction, bit-identical to the reference's
    dataset) fills the same fp32 ring slot on the compute stream before the forward.

    ``score=True``: ``frames`` yields ``(frame, gt_u8)`` pairs, ``gt_u8`` the host uint8 annotations [N,H,W] (pinned
    for real overlap).  The mask crosses on the input stream into a ring slot beside the frame, and ops.davis_measures
    scores the fused map on the compute stream right after the forward; the counts stay on the device until
    ``frame_counts()``.  The results are the same bytes as without scoring."""

    def __init__(self, net, output="logits", depth=3, frames="nchw_f32", meanval=ops.MEANVAL, score=False):
        if output not in ("logits", "bytescale", "prob", "mask"):
            raise ValueError("output must be one of logits / bytescale / prob / mask")
        if frames not in ("nchw_f32", "bgr8"):
            raise ValueError("frames must be nchw_f32 or bgr8")
        self.net, self.output, self.depth = net, output, max(2, int(depth))
        self.frames, self.meanval = frames, tuple(meanval)
        self.score = bool(score)
        self._shape = None
        self._counts = []

    def _allocate(self, shape, device):
        if self.frames == "bgr8":
            n, h, w, _ = shape
            self._dev_raw = [torch.empty(shape, dtype=torch.uint8, device=device) for _ in range(self.depth)]
        else:
            n, _, h, w = shape
        out_dtype = torch.float32 if self.output == "logits" else torch.uint8
        self._dev_in = [torch.empty((n, 3, h, w), dtype=torch.float32, device=device) for _ in range(self.depth)]
        self._dev_out = [torch.empty((n, 1, h, w), dtype=out_dtype, device=device) for _ in range(self.depth)]
        self._host_out = [torch.empty((n, 1, h, w), dtype=out_dtype).pin_memory() for _ in range(self.depth)]
        if self.score:
            self._dev_gt = [torch.empty((n, h, w), dtype=torch.uint8, device=device) for _ in range(self.depth)]
        self._s_in, self._s_out = torch.cuda.Stream(device), torch.cuda.Stream(device)
        mk = lambda: [torch.cuda.Event() for _ in range(self.depth)]
        self._ev_loaded, self._ev_consumed, self._ev_done, self._ev_host = mk(), mk(), mk(), mk()
        self._shape = tuple(shape)
        self.h2d_bytes_per_frame = n * 3 * h * w * (1 if self.frames == "bgr8" else 4) + (n * h * w if self.score else 0)
        self.d2h_bytes_per_frame = n * h * w * (4 if self.output == "logits" else 1)

    def _submit(self, i, frame, gt, device):
        k = i % self.depth
        cur = torch.cuda.current_stream(device)
        bgr8 = self.frames == "bgr8"
        with torch.cuda.stream(self._s_in):
            if i >= self.depth:
                self._s_in.wait_event(self._ev_consumed[k])     # the network has read the previous tenant
            (self._dev_raw[k] if bgr8 else self._dev_in[k]).copy_(frame, non_blocking=True)
            if self.score:
                self._dev_gt[k].copy_(gt, non_blocking=True)
            self._ev_loaded[k].record(self._s_in)
        cur.wait_event(self._ev_loaded[k])
        if i >= self.depth:
            cur.wait_event(self._ev_host[k])                    # previous result of this slot is on the host
        if bgr8:
            # same slot address every time this slot comes round, so the engine's direct graph replay still applies
            ops.image_from_bgr8(self._dev_raw[k], self.meanval, out=self._dev_in[k])
        with torch.no_grad():
            eng = getattr(self.net, "_engine", None)
            if eng is not None:
                # the ring slot is a buffer that comes back: from its second frame on the engine replays a graph captured on
                # the slot itself (no input copy), and the fused map is read out of the graph's static output right here on
                # the same stream (no copy of the five maps into fresh tensors)
                fused = eng.forward(self._dev_in[k], fresh_outputs=False)[-1]
            else:
                fused = self.net(self._dev_in[k])[-1]
            if self.score:
                self._counts.append(ops.davis_measures(fused, self._dev_gt[k]))
            self._ev_consumed[k].record(cur)                    # after the last read of this slot's frame and mask
            if self.output == "logits":
                self._dev_out[k].copy_(fused)
            else:
                ops.logits_to_u8(fused, self.output, out=self._dev_out[k])
        self._ev_done[k].record(cur)
        with torch.cuda.stream(self._s_out):
            self._s_out.wait_event(self._ev_done[k])
            self._host_out[k].copy_(self._dev_out[k], non_blocking=True)
            self._ev_host[k].record(self._s_out)

    def __call__(self, frames):
        device = next(self.net.parameters()).device
        if device.type != "cuda":
            raise RuntimeError("SequenceSegmenter runs on CUDA only; there is no CPU fallback for the OSVOS hot path")
        submitted = 0
        self._counts = []
        with torch.cuda.device(device):
            for item in frames:
                frame, gt = item if self.score else (item, None)
                if frame.dim() == 3:
                    frame = frame.unsqueeze(0)
                if self.score:
                    gt = gt.unsqueeze(0) if gt.dim() == 2 else gt
                    n = frame.shape[0]
                    hw = tuple(frame.shape[1:3]) if self.frames == "bgr8" else tuple(frame.shape[2:4])
                    if gt.dtype != torch.uint8 or tuple(gt.shape) != (n,) + hw:
                        raise ValueError(f"score=True takes uint8 [N,H,W] annotations matching the frames, got "
                                         f"{gt.dtype} {tuple(gt.shape)}")
                if self.frames == "bgr8" and (frame.dtype != torch.uint8 or frame.shape[-1] != 3):
                    raise ValueError("frames='bgr8' takes uint8 [N,H,W,3] frames")
                if self._shape != tuple(frame.shape):
                    if submitted:
                        raise ValueError("all frames of one sequence must share a shape")
                    self._allocate(tuple(frame.shape), device)
                self._submit(submitted, frame, gt, device)
                submitted += 1
                ready = submitted - self.depth + 1              # keep depth-1 frames in flight
                if ready >= 1:
                    k = (ready - 1) % self.depth
                    self._ev_host[k].synchronize()
                    yield self._host_out[k]
            for j in range(max(0, submitted - self.depth + 1), submitted):
                k = j % self.depth
                self._ev_host[k].synchronize()
                yield self._host_out[k]

    def frame_counts(self):
        """int32 [frames*N, 6] host tensor of the last run's ops.davis_measures counts, frame order (score=True);
        one synchronisation."""
        if not self.score:
            raise RuntimeError("frame_counts() needs SequenceSegmenter(..., score=True)")
        if not self._counts:
            return torch.zeros((0, 6), dtype=torch.int32)
        return torch.cat(self._counts).cpu()

    def join_current_stream(self):
        """Make the current stream wait for every copy issued so far (lets CUDA events on the current stream bracket
        the whole pipeline, as bench.py does)."""
        if self._shape is not None:
            cur = torch.cuda.current_stream()
            cur.wait_stream(self._s_in)
            cur.wait_stream(self._s_out)
