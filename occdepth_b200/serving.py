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
uint16 class map [B, X, Y, Z] (4 MB at config 2) and that is what is read back, not the 168 MB of logits.  With
`confidence=True` as well, the float16 top-class probability of every voxel is read back beside it and `result` returns
(map, conf).
"""
import torch

from .engine import require_cuda


def _result_buffers(res):
    """the device and pinned host buffers of one read-back slot: the result's shape, or for a (map, conf) pair one
    uint16 [2, ...] buffer that holds the map and then the confidence's float16 bits"""
    if isinstance(res, tuple):
        dev = torch.empty((2,) + tuple(res[0].shape), dtype=torch.uint16, device=res[0].device)
    else:
        dev = torch.empty_like(res)
    return dev, torch.empty(dev.shape, dtype=dev.dtype).pin_memory()


def _copy_result(dst, res):
    if isinstance(res, tuple):
        dst[0].copy_(res[0])
        dst[1].copy_(res[1].view(torch.uint16))
    else:
        dst.copy_(res)


def _host_result(host, confidence):
    return (host[0], host[1].view(torch.float16)) if confidence else host


class FramePipeline:
    def __init__(self, model, img_shape, pix_shape, fov_shape, device=None, out_key="ssc_logit", classes=False,
                 inv_map=None, confidence=False):
        if not torch.cuda.is_available():
            raise RuntimeError("FramePipeline: occdepth_b200 needs a CUDA (sm_90a) device")
        dev = torch.device(device) if device is not None else next(model.parameters()).device
        require_cuda(torch.empty(0, device=dev), "FramePipeline")
        if confidence and not classes:
            raise ValueError("FramePipeline: confidence=True is the class map's confidence (classes=True)")
        self.model, self.dev, self.out_key = model, dev, out_key
        self.classes, self.inv_map, self.confidence = classes, inv_map, confidence
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
                res = self.model.predict_classes(batch, self.inv_map, confidence=self.confidence)
            else:
                res = self.model(batch)[self.out_key]
        self.in_free[j].record(self.main)
        if self.dev_out[j] is None:
            self.dev_out[j], self.host_out[j] = _result_buffers(res)
        self.main.wait_event(self.out_free[j])
        _copy_result(self.dev_out[j], res)   # the result leaves the allocator-owned tensor on the compute stream
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
        """host tensor of a submitted frame (with `confidence`: (map, conf) views of one pinned buffer); blocks until
        its D2H read has finished.  The buffer is reused by the second submit after the one that produced it."""
        if ticket is None or ticket < self.n - 2 or ticket >= self.n:
            raise ValueError("FramePipeline.result: ticket %r is not one of the two frames in flight" % (ticket,))
        j = ticket & 1
        self.out_free[j].synchronize()
        return _host_result(self.host_out[j], self.confidence)

    def join(self):
        """make the compute stream wait for every outstanding read-back (for timing with CUDA events)"""
        self.main.wait_stream(self.d2h)


class CameraPipeline:
    """`OccDepth.predict_frame` for a stream of camera frames in host memory, with FramePipeline's overlap: the H2D
    copy of frame i+1's uint8 images (and NYU depth map) and the D2H read of frame i-1's class map (or logits) run on
    their own streams while frame i computes.  Per frame only the raw images (3 MB for a KITTI stereo pair), the depth
    PNG and a few matrices leave the host; normalisation, cropping and the projection indices are computed on the
    device, straight into the plan's input buffers.

        pipe = CameraPipeline(model, img_hw=(370, 1220))          # KITTI; geometry fixed per pipeline
        for frame in frames:            # {"img": uint8 (V, H0, W0, 3), "cam_k": (V, 3, 3), "T_velo_2_cam": (V, 4, 4)}
            done = pipe.submit(frame)   # returns the PREVIOUS frame's ticket (or None)
            if done is not None:
                y_pred = pipe.result(done)             # pinned host tensor, valid until two more submits
        y_pred = pipe.result(pipe.flush())

    `frame` is what predict_frame takes (NYU: "img", "cam_pose", "vox_origin", "cam_k", "depth"); the constructor's
    geometry (img_hw, vox_origin, voxel_size, scene_size, pattern_id) fills the keys a frame leaves out.  Two pinned
    and two device image / depth buffers, sized from the first frame and regrown only when a larger raw image arrives;
    nothing else is allocated per frame.  One frame per submit; not for infer_mode with flosp_depth (that route takes
    sampling grids, not camera matrices).

    `confidence=True` (with classes=True) reads back each voxel's float16 top-class probability beside the map into the
    same pinned buffer; `result(ticket)` then returns (map, conf).

    Under enable_slab_parallel (one pipeline per rank, every rank submitting the same frames) `slab_output` is
    required and means what it does for predict_frame: "slab" reads back this rank's X-slab, "root" the whole class
    map (or voxel list) on rank 0 -- the other ranks read nothing back and their `result()` is None.  Under the
    partition's view sharding a rank copies only the view its plan stages (`OccDepth.slab_view`).

    `output="voxels"` lists every frame's occupied voxels on the device (`OccDepth.predict_voxels`) and reads back the
    counts, the class histogram and the first `capacity` rows (flat index, class, voxel centre: 18 bytes a row; default
    capacity an eighth of the output grid) instead of the class map; `result(ticket)` trims them to the rows written
    and says whether the frame held more (`truncated`).  `d2h_bytes` is what a frame reads back.

    `batch=B` runs `OccDepth.predict_frames` instead: `submit` takes a list of 1..B frames, copies them into B-frame
    pinned and device buffers (each frame's slice sized from its own image) and runs the B-frame plan; `result(ticket)`
    returns that submit's n maps [n, X, Y, Z] (or (map, conf)).  A short list -- the last of a stream -- runs the same
    plan, and only its n results are read back.  Not with output="voxels" or slab_output.

    `pixel_format` ("rgb", "bgr" or "nv12") and `rect_maps` (float32 (V, 2, img_h, img_w)) are predict_frame's frame
    keys for every frame that leaves them out: the images are converted and rectified on the device, as OpenCV would on
    the host.  The maps are copied to the device once, here; an NV12 frame copies 1.5 bytes a pixel where RGB copies
    3 (`h2d_bytes`)."""

    def __init__(self, model, img_hw, vox_origin=None, voxel_size=None, scene_size=None, pattern_id=0, classes=True,
                 inv_map=None, device=None, out_key="ssc_logit", output=None, capacity=None, slab_output=None,
                 confidence=False, batch=None, pixel_format="rgb", rect_maps=None):
        if pixel_format not in ("rgb", "bgr", "nv12"):
            raise ValueError("CameraPipeline: pixel_format must be 'rgb', 'bgr' or 'nv12', got %r" % (pixel_format,))
        if batch is not None:
            if isinstance(batch, bool) or not isinstance(batch, int) or batch < 1:
                raise ValueError("CameraPipeline: batch must be None or a frame count >= 1, got %r" % (batch,))
            if output is not None or slab_output is not None:
                raise ValueError("CameraPipeline: batch=%d runs whole class maps (or logits) of unpartitioned plans; "
                                 "output='voxels' and slab_output are not batched" % batch)
        if not torch.cuda.is_available():
            raise RuntimeError("CameraPipeline: occdepth_b200 needs a CUDA (sm_90a) device")
        if output not in (None, "voxels"):
            raise ValueError("CameraPipeline: output must be None (the class map or logits, as `classes` says) or "
                             "'voxels', got %r" % (output,))
        if confidence and (output is not None or not classes):
            raise ValueError("CameraPipeline: confidence=True is the class map's confidence (classes=True, "
                             "output=None); the voxel list has no confidence column")
        if slab_output not in (None, "slab", "root"):
            raise ValueError("CameraPipeline: slab_output must be None, 'slab' or 'root', got %r" % (slab_output,))
        slab = model.__dict__.get("slab_ctx")
        if slab is None:
            if slab_output is not None:
                raise ValueError("CameraPipeline: slab_output=%r needs enable_slab_parallel" % (slab_output,))
        elif slab_output is None:
            raise NotImplementedError("CameraPipeline: under enable_slab_parallel a pipeline needs slab_output='slab' "
                                      "(every rank's X-slab) or 'root' (the whole map on rank 0)")
        if slab_output == "root" and not classes and output is None:
            raise ValueError("CameraPipeline: slab_output='root' gathers the class map (classes=True)")
        if model.infer_mode and model.trans_2d_to_3d == "flosp_depth":
            raise NotImplementedError("CameraPipeline: infer_mode with flosp_depth takes the caller's sampling grids, "
                                      "not camera matrices")
        dev = torch.device(device) if device is not None else next(model.parameters()).device
        require_cuda(torch.empty(0, device=dev), "CameraPipeline")
        self.model, self.dev, self.out_key = model, dev, out_key
        self.classes, self.inv_map, self.confidence = classes, inv_map, confidence
        self.geometry = {"img_hw": tuple(img_hw), "pattern_id": int(pattern_id)}
        for k, v in (("vox_origin", vox_origin), ("voxel_size", voxel_size), ("scene_size", scene_size)):
            if v is not None:
                self.geometry[k] = v
        if pixel_format != "rgb":
            self.geometry["pixel_format"] = pixel_format
        if rect_maps is not None:
            import numpy as np
            maps = torch.as_tensor(np.ascontiguousarray(rect_maps) if not isinstance(rect_maps, torch.Tensor)
                                   else rect_maps)
            if maps.dtype != torch.float32 or maps.dim() != 4 or tuple(maps.shape[1:]) != (2,) + tuple(img_hw):
                raise ValueError("CameraPipeline: rect_maps must be float32 (V, 2, %d, %d)" % tuple(img_hw))
            self.geometry["rect_maps"] = maps.to(dev).contiguous()
        self.main = torch.cuda.current_stream(dev)
        self.h2d, self.d2h = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        self.bufs = {}                # name -> two (pinned host, device) flat byte buffers
        self.batch = batch
        self.counts = [0, 0]          # batch: the frames each result buffer holds
        self.dev_out, self.host_out = [None, None], [None, None]
        self.in_ready, self.in_free, self.host_free, self.out_ready, self.out_free = (
            [torch.cuda.Event(), torch.cuda.Event()] for _ in range(5))
        for j in range(2):
            self.in_free[j].record(self.main)
            self.host_free[j].record(self.h2d)
            self.out_free[j].record(self.main)
        self.n = 0
        self.h2d_bytes = 0            # bytes copied host -> device by the last submit
        self.output = output
        self.slab_output = slab_output
        self.reads_back = slab_output != "root" or slab.rank == 0     # "root": only rank 0 has a result
        if output == "voxels":
            n_out = 1
            for s in model.full_scene_size:
                n_out *= int(s)
            self.capacity = n_out // 8 if capacity is None else int(capacity)
            self.vox = [None, None]       # the two device lists, overwritten in place
            self.d2h_bytes = 0            # bytes read back per frame

    @staticmethod
    def _host(x, what):
        if isinstance(x, torch.Tensor):
            if x.is_cuda:
                raise ValueError("CameraPipeline.submit: frame[%r] must be in host memory" % what)
            return x
        import numpy as np
        return torch.from_numpy(np.ascontiguousarray(x))

    def _stage_h2d(self, name, j, x):
        """copy host tensor x into pinned buffer j (once its previous H2D has finished), enqueue the H2D copy into
        device buffer j; returns the device view of x's shape"""
        nb = x.numel() * x.element_size()
        buf = self.bufs.setdefault(name, [None, None])[j]
        if buf is None or buf[0].numel() < nb:
            torch.cuda.synchronize(self.dev)      # a larger raw image: nothing may still read the old buffers
            buf = (torch.empty(nb, dtype=torch.uint8).pin_memory(), torch.empty(nb, dtype=torch.uint8, device=self.dev))
            self.bufs[name][j] = buf
        host = buf[0][:nb].view(x.dtype).view(x.shape)
        host.copy_(x)
        dev = buf[1][:nb].view(x.dtype).view(x.shape)
        dev.copy_(host, non_blocking=True)        # on the h2d stream (the caller's context)
        self.h2d_bytes += nb
        return dev

    def submit(self, frame):
        """enqueue one camera frame (host arrays / tensors, see the class docstring), or with `batch` a list of 1..B
        frames.  Returns the ticket of the submit before this one -- its read-back overlaps this one's forward -- or
        None."""
        if self.batch is not None:
            return self._submit_batch(frame)
        img = self._host(frame["img"], "img")
        if img.dim() == 5:
            if img.shape[0] != 1:
                raise NotImplementedError("CameraPipeline.submit: one frame per submit (batch size %d)" % img.shape[0])
            img = img[0]
        if frame.get("pixel_format", self.geometry.get("pixel_format")) == "nv12":
            img = img.unsqueeze(0) if img.dim() == 2 else img          # (V, H0 * 3 / 2, W0)
        elif img.dim() == 3:
            img = img.unsqueeze(0)                                     # (V, H0, W0, 3)
        depth = frame.get("depth")
        depth = None if depth is None else self._host(depth, "depth")
        V = int(img.shape[0])
        sel = self.model.slab_view(V, virtual=depth is not None)
        j = self.n & 1
        self.host_free[j].synchronize()           # pinned buffer j: its previous H2D copy has been read
        self.h2d_bytes = 0
        f = dict(self.geometry)
        f.update(frame)
        with torch.cuda.stream(self.h2d):
            self.h2d.wait_event(self.in_free[j])
            if sel is None:
                f["img"] = self._stage_h2d("img", j, img)
            else:
                # this rank's plan stages view `sel` only: copy that one, and let every view of the frame read it
                f["img"] = self._stage_h2d("img", j, img[sel:sel + 1]).expand((V,) + tuple(img.shape[1:]))
            if depth is not None:
                f["depth"] = self._stage_h2d("depth", j, depth)
            self.in_ready[j].record(self.h2d)
            self.host_free[j].record(self.h2d)
        self.main.wait_event(self.in_ready[j])
        if self.output == "voxels":
            return self._submit_voxels(f, j)
        with torch.no_grad():
            res = self.model.predict_frame(f, classes=self.classes, inv_map=self.inv_map,
                                           slab_output=self.slab_output, confidence=self.confidence)
        self.in_free[j].record(self.main)
        if not self.reads_back:
            self.n += 1
            return self.n - 2 if self.n >= 2 else None
        if not self.classes:
            res = res[self.out_key]
        shape = (2,) + tuple(res[0].shape) if self.confidence else res.shape
        if self.dev_out[j] is None or self.dev_out[j].shape != shape:
            self.out_free[j].synchronize()
            self.dev_out[j], self.host_out[j] = _result_buffers(res)
        self.main.wait_event(self.out_free[j])
        _copy_result(self.dev_out[j], res)   # the result leaves the allocator-owned tensor on the compute stream
        self.out_ready[j].record(self.main)
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(self.out_ready[j])
            self.host_out[j].copy_(self.dev_out[j], non_blocking=True)
            self.out_free[j].record(self.d2h)
        self.n += 1
        return self.n - 2 if self.n >= 2 else None

    def _submit_batch(self, frames):
        """submit for batch=B: the frames' images (and depth maps) into slot j's per-item buffers, predict_frames'
        B-frame plan, and the read-back of the first n results"""
        m = self.model
        fs = [dict(self.geometry, **fr) for fr in frames] if isinstance(frames, (list, tuple)) else frames
        m._frames_checked(fs, self.classes, self.confidence, batch=self.batch, inputs=False)   # nothing moved yet
        n = len(fs)
        j = self.n & 1
        self.host_free[j].synchronize()           # pinned buffers j: their previous H2D copies have been read
        self.h2d_bytes = 0
        with torch.cuda.stream(self.h2d):
            self.h2d.wait_event(self.in_free[j])
            for i, f in enumerate(fs):
                img = self._host(f["img"], "img")
                if img.dim() == 5:
                    if img.shape[0] != 1:
                        raise NotImplementedError("CameraPipeline.submit: frame %d holds %d frames; give one dict per "
                                                  "frame" % (i, img.shape[0]))
                    img = img[0]
                f["img"] = self._stage_h2d("img%d" % i, j, img)
                if f.get("depth") is not None:
                    f["depth"] = self._stage_h2d("depth%d" % i, j, self._host(f["depth"], "depth"))
            self.in_ready[j].record(self.h2d)
            self.host_free[j].record(self.h2d)
        self.main.wait_event(self.in_ready[j])
        with torch.no_grad():
            res = m._run_frames([m._frame_checked(f, None, self.classes) for f in fs], self.batch, self.classes,
                                self.inv_map, self.confidence)
        self.in_free[j].record(self.main)
        if not self.classes:
            res = res[self.out_key]
        parts = list(res) if self.confidence else [res]
        shape = (len(parts), self.batch) + tuple(parts[0].shape[1:])
        if self.dev_out[j] is None or tuple(self.dev_out[j].shape) != shape:
            self.out_free[j].synchronize()
            self.dev_out[j] = torch.empty(shape, dtype=torch.uint16 if self.classes else parts[0].dtype,
                                          device=self.dev)
            self.host_out[j] = torch.empty(shape, dtype=self.dev_out[j].dtype).pin_memory()
        self.main.wait_event(self.out_free[j])
        for k, p in enumerate(parts):   # the results leave the allocator-owned tensors on the compute stream
            self.dev_out[j][k, :n].copy_(p.view(torch.uint16) if p.dtype == torch.float16 else p)
        self.out_ready[j].record(self.main)
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(self.out_ready[j])
            for k in range(len(parts)):
                self.host_out[j][k, :n].copy_(self.dev_out[j][k, :n], non_blocking=True)
            self.out_free[j].record(self.d2h)
        self.counts[j] = n
        self.n += 1
        return self.n - 2 if self.n >= 2 else None

    def _submit_voxels(self, f, j):
        """the tail of submit for output="voxels": list the frame into device list j, then read back the counts, the
        histogram and the first `capacity` rows in one batch of copies -- the host learns the count from that same
        batch, so no second round trip decides how much to copy"""
        self.main.wait_event(self.out_free[j])        # list j is overwritten in place: its last read-back is done
        with torch.no_grad():
            vl = self.model.predict_voxels(f, inv_map=self.inv_map, capacity=self.capacity, out=self.vox[j],
                                           slab_output=self.slab_output)
        self.in_free[j].record(self.main)
        if not self.reads_back:
            self.n += 1
            return self.n - 2 if self.n >= 2 else None
        if self.vox[j] is None:
            self.vox[j] = vl
            self.host_out[j] = {k: torch.empty(getattr(vl, k)[0].shape, dtype=getattr(vl, k).dtype).pin_memory()
                                for k in ("count", "hist", "index", "cls", "xyz")}
            self.d2h_bytes = sum(t.numel() * t.element_size() for t in self.host_out[j].values())
        self.out_ready[j].record(self.main)
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(self.out_ready[j])
            for k, host in self.host_out[j].items():
                host.copy_(getattr(vl, k)[0], non_blocking=True)
            self.out_free[j].record(self.d2h)
        self.n += 1
        return self.n - 2 if self.n >= 2 else None

    def flush(self):
        """ticket of the last submitted frame (nothing further overlaps its read-back)"""
        return self.n - 1 if self.n else None

    def result(self, ticket):
        """host tensor (pinned) of a submitted frame, or with `confidence` (map, conf) views of one pinned buffer;
        blocks until its D2H read has finished.  The buffer is reused by
        the second submit after the one that produced it.  With output="voxels": a dict of numpy views of the pinned
        buffers, trimmed to the rows that were written -- "count" (inside, outside the FOV; the true counts), "hist",
        "index", "cls", "xyz" (the in-FOV rows first, "n_in" of them) and "truncated".  None on a rank other than 0
        with slab_output="root"."""
        if ticket is None or ticket < self.n - 2 or ticket >= self.n:
            raise ValueError("CameraPipeline.result: ticket %r is not one of the two frames in flight" % (ticket,))
        if not self.reads_back:
            return None
        j = ticket & 1
        self.out_free[j].synchronize()
        if self.batch is not None:
            h = self.host_out[j][:, :self.counts[j]]
            return (h[0], h[1].view(torch.float16)) if self.confidence else h[0]
        if self.output == "voxels":
            h = {k: v.numpy() for k, v in self.host_out[j].items()}
            count = h["count"].astype("int64")
            total = int(count.sum())
            n = min(total, self.capacity)
            return dict(count=count, hist=h["hist"], index=h["index"][:n], cls=h["cls"][:n], xyz=h["xyz"][:n],
                        n_in=min(int(count[0]), n), truncated=total > self.capacity)
        return _host_result(self.host_out[j], self.confidence)

    def join(self):
        """make the compute stream wait for every outstanding read-back (for timing with CUDA events)"""
        self.main.wait_stream(self.d2h)
