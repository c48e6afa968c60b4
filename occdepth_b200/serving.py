"""Frame pipeline around `OccDepth.forward` for callers that hold their frames in HOST memory (the reference's
`eval.py` / `scripts/generate_output.py` loops: `model(batch)` then `.cpu()` on the logits, generate_output.py:94-97).

One forward of config 2 moves 21 MB of inputs in and 168 MB of logits out over PCIe; run back to back with the
forward, those copies add their whole duration to every frame.  `FramePipeline` keeps two
pre-allocated input and output buffer sets on the device and two pinned result buffers on the host, and issues the
H2D copy of frame i+1 and the D2H read of frame i-1 on their own copy streams while frame i computes.  Nothing is
allocated per frame (a caching-allocator block that changes streams would serialise them again).

    pipe = FramePipeline(model, img_shape, pix_shape, fov_shape)
    for frame in frames:                       # pinned host tensors
        done = pipe.submit(frame.img, frame.pix, frame.fov)   # returns the PREVIOUS frame's ticket (or None)
        if done is not None:
            logits = pipe.result(done)         # host tensor, valid until two more submits
    logits = pipe.result(pipe.flush())

With `classes=True` every frame runs `model.predict_classes(batch, inv_map)` instead: the classifier writes the
uint16 class map [B, X, Y, Z] (4 MB at config 2) and that is what is read back, not the 168 MB of logits.
"""
import torch

from .engine import require_cuda


class FramePipeline:
    def __init__(self, model, img_shape, pix_shape, fov_shape, device=None, out_key="ssc_logit", classes=False,
                 inv_map=None):
        if not torch.cuda.is_available():
            raise RuntimeError("FramePipeline: occdepth_b200 needs a CUDA (sm_90a) device")
        dev = torch.device(device) if device is not None else next(model.parameters()).device
        require_cuda(torch.empty(0, device=dev), "FramePipeline")
        self.model, self.dev, self.out_key = model, dev, out_key
        self.classes, self.inv_map = classes, inv_map
        self.key = "%d" % model.project_scale
        self.main = torch.cuda.current_stream(dev)
        self.h2d, self.d2h = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        self.dev_in = [{"img": torch.empty(img_shape, dtype=torch.float32, device=dev),
                        "pix": torch.empty(pix_shape, dtype=torch.int64, device=dev),
                        "fov": torch.empty(fov_shape, dtype=torch.bool, device=dev)} for _ in range(2)]
        self.dev_out = [None, None]          # allocated on the first forward (the output shape is the model's)
        self.host_out = [None, None]
        self.in_ready, self.in_free, self.out_ready, self.out_free = (
            [torch.cuda.Event(), torch.cuda.Event()] for _ in range(4))
        for j in range(2):
            self.in_free[j].record(self.main)
            self.out_free[j].record(self.main)
        self.n = 0

    def submit(self, img_h, pix_h, fov_h):
        """enqueue one frame (pinned host tensors; pageable ones work but their copies block the host).  Returns the
        ticket of the frame submitted before this one -- its read-back overlaps this frame's forward -- or None."""
        j = self.n & 1
        buf = self.dev_in[j]
        with torch.cuda.stream(self.h2d):
            self.h2d.wait_event(self.in_free[j])
            buf["img"].copy_(img_h, non_blocking=True)
            buf["pix"].copy_(pix_h, non_blocking=True)
            buf["fov"].copy_(fov_h, non_blocking=True)
            self.in_ready[j].record(self.h2d)
        self.main.wait_event(self.in_ready[j])
        batch = {"img": buf["img"], "projected_pix_" + self.key: [buf["pix"]], "fov_mask_" + self.key: [buf["fov"]]}
        with torch.no_grad():
            if self.classes:
                res = self.model.predict_classes(batch, self.inv_map)
            else:
                res = self.model(batch)[self.out_key]
        self.in_free[j].record(self.main)
        if self.dev_out[j] is None:
            self.dev_out[j] = torch.empty_like(res)
            self.host_out[j] = torch.empty(res.shape, dtype=res.dtype).pin_memory()
        self.main.wait_event(self.out_free[j])
        self.dev_out[j].copy_(res)           # the result leaves the allocator-owned tensor on the compute stream
        self.out_ready[j].record(self.main)
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(self.out_ready[j])
            self.host_out[j].copy_(self.dev_out[j], non_blocking=True)
            self.out_free[j].record(self.d2h)
        self.n += 1
        return self.n - 2 if self.n >= 2 else None

    def flush(self):
        """ticket of the last submitted frame (nothing further overlaps its read-back)"""
        return self.n - 1 if self.n else None

    def result(self, ticket):
        """host tensor of a submitted frame; blocks until its D2H read has finished.  The buffer is reused by the
        second submit after the one that produced it."""
        if ticket is None or ticket < self.n - 2 or ticket >= self.n:
            raise ValueError("FramePipeline.result: ticket %r is not one of the two frames in flight" % (ticket,))
        j = ticket & 1
        self.out_free[j].synchronize()
        return self.host_out[j]

    def join(self):
        """make the compute stream wait for every outstanding read-back (for timing with CUDA events)"""
        self.main.wait_stream(self.d2h)
