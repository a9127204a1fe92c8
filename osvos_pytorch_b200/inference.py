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
    ``frame_counts()``.  The results are the same bytes as without scoring.

    ``input_res`` (``frames="bgr8"`` only): the reference's ``inputRes`` (davis.imresize_size).  Each slot's bytes are
    resized on the compute stream (ops.resize_u8, bilinear; the mask nearest) into a resized slot of fixed address
    before the float conversion, so the network, the results and the scores are at that size, as the reference's test
    loop writes them.

    ``output_res="stored"`` (with ``input_res``): each fused map is resized back to the frames' stored size on the
    compute stream (ops.resize_f32, scipy 1.0's imresize(mode='F'); DESIGN.md §18) into a per-slot buffer of fixed
    address, so the results are [N,1,H0,W0] and the scores are taken against the original annotations, as the
    DAVIS-2016 benchmark scores 480x854 masks.  ``"network"`` (the default) keeps them at the network resolution.
    Without ``input_res`` both are the stored size and nothing is resized.

    ``frames="jpeg"``: ``frames`` yields collated batches (davis.collate) of a DAVIS2016Frames(decode="device")
    dataset; with ``score=True`` their masks are the annotations (no pairs).  Each batch's buffer crosses PCIe into a
    per-slot device buffer (grown when a larger batch arrives: the decode is not captured in a graph, only the
    forward on the fp32 slot is), and the JPEGs are decoded on the compute stream into the slot's bgr8 buffer; from
    there on it is ``frames="bgr8"``.  ``jpeg_status`` (int32 [1] on the device) sums the decoder's status words
    over the run: nonzero when a stream was corrupt or cut short.

    ``encode="png"`` (``output`` bytescale / prob / mask): each uint8 result is encoded on the compute stream
    (ops.encode_png, DESIGN.md §21) into a per-slot buffer of fixed address, and the whole buffer (the per-frame
    capacity, so no size is read back first) and the file lengths cross device->host instead of the maps.  Each result
    is then a list of N ``memoryview``s, each one complete PNG file (what Image.fromarray(map, "L").save writes, other
    deflate bytes) backed by the pinned slot and valid as long as the maps are without it.

    ``overlay="jpeg"`` (``frames="bgr8"`` or ``"jpeg"``): each frame's mask drawn over its bytes (ops.overlay_mask: the
    frame at the results' size, i.e. the resized slot under ``input_res`` or the stored bytes under
    ``output_res="stored"``, and the fused map after any resize) and encoded as the JPEG cv2.imencode would write at
    ``overlay_quality`` (ops.encode_jpeg, DESIGN.md §23), on the compute stream before the slot is released, into a
    per-slot buffer of fixed address that crosses device->host at its capacity with the file lengths.  Each yielded
    item is then ``(result, overlays)``, ``overlays`` a list of N ``memoryview``s, one complete JPEG file each, valid
    as long as the result is.

    ``nets=[net_1, ..., net_K]`` with ``output="labels"`` (DAVIS-2017, one fine-tuned network per object; DESIGN.md
    §24): per frame every net's forward runs on the same fp32 slot and ops.merge_objects turns the K fused maps into
    the slot's uint8 label map (1 + the object of the largest positive logit, 0 background), so each result is uint8
    [N,1,H,W] of object ids.  ``score=True`` scores it with ops.davis_measures_objects against the slot's annotation
    (object ids, 255 void) and ``frame_counts()`` returns [frames*N, K, 6].  ``encode="png"`` with ``palette`` (the
    PLTE bytes, e.g. the first annotation's) writes palette files.  With ``input_res`` labels need
    ``output_res="stored"`` (DESIGN.md §27): the K forwards run on the resized slot and ops.upsample_merge_objects
    writes the stored-size label map straight from the K fused maps (each upsampled as ops.resize_f32 does, then
    merged; an argmax cannot be upsampled after the merge), so results, scores against the original annotations and
    palette files are at the stored size.  A label map at the network resolution is not what the DAVIS-2017 toolkit
    scores, so labels with ``input_res`` and ``output_res="network"`` are refused, as is ``overlay`` with labels."""

    def __init__(self, net=None, output="logits", depth=3, frames="nchw_f32", meanval=ops.MEANVAL, score=False,
                 input_res=None, output_res="network", encode=None, overlay=None, overlay_quality=95, nets=None,
                 palette=None):
        if (net is None) == (nets is None):
            raise ValueError("pass either net or nets")
        nets = [net] if nets is None else list(nets)
        if not 1 <= len(nets) <= 254 or len({id(m) for m in nets}) != len(nets):
            raise ValueError("nets must be 1 .. 254 distinct networks")
        if output not in ("logits", "bytescale", "prob", "mask", "labels"):
            raise ValueError("output must be one of logits / bytescale / prob / mask / labels")
        if len(nets) > 1 and output != "labels":
            raise ValueError("several nets are merged into a label map: they need output='labels'")
        if output == "labels" and ((input_res is not None and output_res != "stored") or overlay is not None):
            raise ValueError("output='labels' writes label maps at the stored size: with input_res it needs "
                             "output_res='stored', and it does not take overlay")
        if palette is not None and (output != "labels" or encode != "png"):
            raise ValueError("palette writes label maps as palette PNGs: it needs output='labels' and encode='png'")
        if frames not in ("nchw_f32", "bgr8", "jpeg"):
            raise ValueError("frames must be nchw_f32, bgr8 or jpeg")
        if input_res is not None and frames == "nchw_f32":
            raise ValueError("input_res resizes the decoded bytes, as imresize does: it needs frames='bgr8' or 'jpeg'")
        if output_res not in ("network", "stored"):
            raise ValueError("output_res must be 'network' or 'stored'")
        if encode not in (None, "png"):
            raise ValueError("encode must be None or 'png'")
        if encode == "png" and output == "logits":
            raise ValueError("encode='png' writes 8-bit maps: it needs output bytescale, prob or mask")
        if overlay not in (None, "jpeg"):
            raise ValueError("overlay must be None or 'jpeg'")
        if overlay == "jpeg" and frames == "nchw_f32":
            raise ValueError("overlay='jpeg' draws over the frames' bytes: it needs frames='bgr8' or 'jpeg'")
        if not 1 <= int(overlay_quality) <= 100:
            raise ValueError("overlay_quality must lie in 1..100")
        self.nets, self.net, self.output, self.depth = nets, nets[0], output, max(2, int(depth))
        self.palette = None if palette is None else bytes(palette)
        self.frames, self.meanval = frames, tuple(meanval)
        self.score = bool(score)
        self.input_res = input_res
        self.output_res = output_res
        self._upsample = input_res is not None and output_res == "stored"
        self.encode = encode
        self.overlay, self.overlay_quality = overlay, int(overlay_quality)
        self._shape = None
        self._counts = []
        self.jpeg_status = None

    def _allocate(self, shape, device):
        if self.frames != "nchw_f32":
            n, h, w, _ = shape
            self._dev_blob = [None] * self.depth
            self._dev_raw = [torch.empty(shape, dtype=torch.uint8, device=device) for _ in range(self.depth)]
        else:
            n, _, h, w = shape
        h0, w0 = h, w
        if self.input_res is not None:
            from .davis import imresize_size
            h, w = imresize_size(self.input_res, h0, w0)
            self._dev_rs = [torch.empty((n, h, w, 3), dtype=torch.uint8, device=device) for _ in range(self.depth)]
        out_dtype = torch.float32 if self.output == "logits" else torch.uint8
        rh, rw = (h0, w0) if self._upsample else (h, w)                  # the results' size
        self._dev_in = [torch.empty((n, 3, h, w), dtype=torch.float32, device=device) for _ in range(self.depth)]
        self._dev_out = [torch.empty((n, 1, rh, rw), dtype=out_dtype, device=device) for _ in range(self.depth)]
        if self.encode == "png":
            cap = ops.png_max_bytes(rh, rw, self.palette)
            self._dev_png = [torch.empty((n, cap), dtype=torch.uint8, device=device) for _ in range(self.depth)]
            self._dev_len = [torch.empty(n, dtype=torch.int64, device=device) for _ in range(self.depth)]
            self._host_png = [torch.empty((n, cap), dtype=torch.uint8).pin_memory() for _ in range(self.depth)]
            self._host_len = [torch.empty(n, dtype=torch.int64).pin_memory() for _ in range(self.depth)]
        else:
            self._host_out = [torch.empty((n, 1, rh, rw), dtype=out_dtype).pin_memory() for _ in range(self.depth)]
        if self.overlay == "jpeg":
            ocap = ops.jpeg_max_bytes(rh, rw)
            self._dev_ovl = torch.empty((n, rh, rw, 3), dtype=torch.uint8, device=device)   # compute stream only
            self._dev_jpg = [torch.empty((n, ocap), dtype=torch.uint8, device=device) for _ in range(self.depth)]
            self._dev_jlen = [torch.empty(n, dtype=torch.int64, device=device) for _ in range(self.depth)]
            self._host_jpg = [torch.empty((n, ocap), dtype=torch.uint8).pin_memory() for _ in range(self.depth)]
            self._host_jlen = [torch.empty(n, dtype=torch.int64).pin_memory() for _ in range(self.depth)]
        if self._upsample and self.output != "labels":     # labels are upsampled inside the merge
            self._dev_up = [torch.empty((n, 1, h0, w0), dtype=torch.float32, device=device) for _ in range(self.depth)]
        if self.score:
            self._dev_gt = [torch.empty((n, h0, w0), dtype=torch.uint8, device=device) for _ in range(self.depth)]
            if self.input_res is not None and not self._upsample:
                self._dev_gt_rs = [torch.empty((n, h, w), dtype=torch.uint8, device=device) for _ in range(self.depth)]
        self._s_in, self._s_out = torch.cuda.Stream(device), torch.cuda.Stream(device)
        mk = lambda: [torch.cuda.Event() for _ in range(self.depth)]
        self._ev_loaded, self._ev_consumed, self._ev_done, self._ev_host = mk(), mk(), mk(), mk()
        self._shape = tuple(shape)
        self.h2d_bytes_per_frame = n * 3 * h0 * w0 * (4 if self.frames == "nchw_f32" else 1) + (n * h0 * w0 if self.score else 0)
        self.d2h_bytes_per_frame = n * rh * rw * (4 if self.output == "logits" else 1)
        if self.encode == "png":
            self.d2h_bytes_per_frame = n * (cap + 8)
        if self.overlay == "jpeg":
            self.d2h_bytes_per_frame += n * (ocap + 8)

    def _submit(self, i, frame, gt, device):
        k = i % self.depth
        cur = torch.cuda.current_stream(device)
        bgr8 = self.frames != "nchw_f32"
        jpeg = self.frames == "jpeg"
        with torch.cuda.stream(self._s_in):
            if i >= self.depth:
                self._s_in.wait_event(self._ev_consumed[k])     # the network has read the previous tenant
            if jpeg:                                            # the collated buffer: JPEGs, fallback frames, masks
                from .davis import pinned
                data = pinned(frame["data"])
                if self._dev_blob[k] is None or self._dev_blob[k].numel() < data.numel():
                    self._dev_blob[k] = torch.empty(data.numel(), dtype=torch.uint8, device=device)
                self._dev_blob[k][:data.numel()].copy_(data, non_blocking=True)
                self.h2d_bytes_per_frame = data.numel()
            else:
                (self._dev_raw[k] if bgr8 else self._dev_in[k]).copy_(frame, non_blocking=True)
            if self.score and not jpeg:
                self._dev_gt[k].copy_(gt, non_blocking=True)
            self._ev_loaded[k].record(self._s_in)
        cur.wait_event(self._ev_loaded[k])
        if i >= self.depth:
            cur.wait_event(self._ev_host[k])                    # previous result of this slot is on the host
        gt_dev = self._dev_gt[k] if self.score else None
        if jpeg:
            from .davis import _assemble, views
            n, h, w = (int(v) for v in frame["size"])
            blob = self._dev_blob[k][:frame["data"].numel()]
            if "jpeg" in frame:
                _, gt_view, _ = _assemble(blob, frame["jpeg"], n, h, w, self.jpeg_status, out=self._dev_raw[k])
            else:                                               # every frame of the batch fell back to cv2.imread
                img_view, gt_view = views(blob, n, h, w)
                self._dev_raw[k].copy_(img_view)
            if self.score:
                gt_dev = gt_view
        if bgr8:
            raw = self._dev_raw[k]
            if self.input_res is not None:
                raw = ops.resize_u8(raw, self._dev_rs[k].shape[1:3], "bilinear", out=self._dev_rs[k])
                if self.score and not self._upsample:
                    gt_dev = ops.resize_u8(gt_dev, self._dev_gt_rs[k].shape[1:3], "nearest", out=self._dev_gt_rs[k])
            # same slot address every time this slot comes round, so the engine's direct graph replay still applies
            ops.image_from_bgr8(raw, self.meanval, out=self._dev_in[k])
        with torch.no_grad():
            fused_maps = []
            for net in self.nets:
                eng = getattr(net, "_engine", None)
                if eng is not None:
                    # the ring slot is a buffer that comes back: from its second frame on the engine replays a graph
                    # captured on the slot itself (no input copy), and the fused map is read out of the graph's static
                    # output right here on the same stream (no copy of the five maps into fresh tensors); each net has
                    # its own engine, so the K static outputs stay valid until the merge below
                    fused_maps.append(eng.forward(self._dev_in[k], fresh_outputs=False)[-1])
                else:
                    fused_maps.append(net(self._dev_in[k])[-1])
            fused = fused_maps[0]
            if self._upsample and self.output != "labels":     # back to the stored size, before anything reads it
                fused = ops.resize_f32(fused, self._dev_up[k].shape[2:4], out=self._dev_up[k])
            if self.output == "labels":
                if self._upsample:                              # each object's map upsampled, then merged
                    labels = ops.upsample_merge_objects(fused_maps, self._dev_out[k].shape[2:4], out=self._dev_out[k])
                else:
                    labels = ops.merge_objects(fused_maps, out=self._dev_out[k])
                if self.score:
                    self._counts.append(ops.davis_measures_objects(labels, gt_dev, len(self.nets)))
            elif self.score:
                self._counts.append(ops.davis_measures(fused, gt_dev))
            if self.overlay == "jpeg":                          # reads the slot's frame: before the slot is released
                img = ops.overlay_mask(self._dev_raw[k] if self._upsample else raw, fused, out=self._dev_ovl)
                ops.encode_jpeg(img, self.overlay_quality, out=self._dev_jpg[k], lengths=self._dev_jlen[k])
            self._ev_consumed[k].record(cur)                    # after the last read of this slot's frame and mask
            if self.output == "logits":
                self._dev_out[k].copy_(fused)
            else:
                if self.output != "labels":
                    ops.logits_to_u8(fused, self.output, out=self._dev_out[k])
                if self.encode == "png":
                    ops.encode_png(self._dev_out[k], out=self._dev_png[k], lengths=self._dev_len[k], palette=self.palette)
        self._ev_done[k].record(cur)
        with torch.cuda.stream(self._s_out):
            self._s_out.wait_event(self._ev_done[k])
            if self.encode == "png":
                self._host_png[k].copy_(self._dev_png[k], non_blocking=True)
                self._host_len[k].copy_(self._dev_len[k], non_blocking=True)
            else:
                self._host_out[k].copy_(self._dev_out[k], non_blocking=True)
            if self.overlay == "jpeg":
                self._host_jpg[k].copy_(self._dev_jpg[k], non_blocking=True)
                self._host_jlen[k].copy_(self._dev_jlen[k], non_blocking=True)
            self._ev_host[k].record(self._s_out)

    def _result(self, k):
        self._ev_host[k].synchronize()
        if self.encode != "png":
            res = self._host_out[k]
        else:
            files = self._host_png[k].numpy()
            res = [memoryview(files[j, :int(ln)]) for j, ln in enumerate(self._host_len[k].tolist())]
        if self.overlay != "jpeg":
            return res
        files = self._host_jpg[k].numpy()
        return res, [memoryview(files[j, :int(ln)]) for j, ln in enumerate(self._host_jlen[k].tolist())]

    def __call__(self, frames):
        device = next(self.net.parameters()).device
        if device.type != "cuda":
            raise RuntimeError("SequenceSegmenter runs on CUDA only; there is no CPU fallback for the OSVOS hot path")
        submitted = 0
        self._counts = []
        with torch.cuda.device(device):
            if self.frames == "jpeg":
                self.jpeg_status = torch.zeros(1, dtype=torch.int32, device=device)
            for item in frames:
                if self.frames == "jpeg":
                    n, h, w = (int(v) for v in item["size"])
                    if self._shape != (n, h, w, 3):
                        if submitted:
                            raise ValueError("all frames of one sequence must share a shape")
                        self._allocate((n, h, w, 3), device)
                    self._submit(submitted, item, None, device)
                    submitted += 1
                    ready = submitted - self.depth + 1
                    if ready >= 1:
                        k = (ready - 1) % self.depth
                        yield self._result(k)
                    continue
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
                    yield self._result(k)
            for j in range(max(0, submitted - self.depth + 1), submitted):
                k = j % self.depth
                yield self._result(k)

    def frame_counts(self):
        """int32 [frames*N, 6] host tensor of the last run's ops.davis_measures counts, frame order (score=True);
        [frames*N, K, 6] of ops.davis_measures_objects with output="labels".  One synchronisation."""
        if not self.score:
            raise RuntimeError("frame_counts() needs SequenceSegmenter(..., score=True)")
        if not self._counts:
            return torch.zeros((0, len(self.nets), 6) if self.output == "labels" else (0, 6), dtype=torch.int32)
        return torch.cat(self._counts).cpu()

    def join_current_stream(self):
        """Make the current stream wait for every copy issued so far (lets CUDA events on the current stream bracket
        the whole pipeline, as bench.py does)."""
        if self._shape is not None:
            cur = torch.cuda.current_stream()
            cur.wait_stream(self._s_in)
            cur.wait_stream(self._s_out)
