"""FaceAnaImages — FaceAna.run for many still images per call (additive API, SURVEY.md 8b).

The reference analyses a folder of photos with `facer.run(image); facer.reset()` per image (demo.py images()).  Here one
call takes any number of images of any sizes, host arrays or CUDA tensors, and runs the detector in batches of
max_frames and the landmark net in batches of max_faces on exactly the faces found:

    fi = FaceAnaImages(top_k=16)
    res = fi.run_batch(images)          # one list of {'box','kps','scores'} per image, what FaceAna.run returns after reset()
    fi = FaceAnaImages(top_k=16, align=112)     # also 'chip' and 'M' per face, as FaceAna(align=112) returns them
    # overlapped: while one call's landmarks run, the next call stages its images
    fi.submit(images_0); fi.submit(images_1); r0 = fi.collect(); fi.submit(images_2); r1 = fi.collect(); ...
    # CUDA images, results left on the GPU, packed by image:
    out = fi.new_results(len(cuda_images)); fi.submit(cuda_images, out=out); fi.collect()

One call on the GPU: FaceDetector's batched letterbox, network and NMS; skps_select_faces_batch (sort_and_filter with no
track boxes, one block per image); one read-back of the face counts and selected boxes, which size the landmark batch and,
for host images, cut their upload to the crop rectangles; FaceLandmark's batched crops, network and de-normalisation;
skps_landmark_boxes (the returned box, judge_boxs(boxes, rects(kps))); with pose, skps_head_pose_faces.  With align,
FaceLandmark's chip stage: skps_align_estimate right after the landmarks, and skps_warp_faces on CUDA images there too, or
on the rectangles of host images each chip reads at collect().
"""
import numpy as np

from ... import runtime as rt
from ...graph_tools import check_detector_input
from .align import check_size
from .face_detector import FaceDetector
from .face_landmark import FaceLandmark
from .facer import MAX_TOP_K, get_cfg
from .staging import check_frames, check_out, grow, new_buffers, pad16

POSE_FIELDS = (("rvec", (3,)), ("tvec", (3,)), ("euler", (3,)), ("reproject", (8, 2)))


def pack_faces(counts):
    """The packing of a call's faces: counts[i] faces of image i, in image order.  Returns (first, face_image) as int32
    arrays: image i's faces are rows first[i] .. first[i] + counts[i] - 1, and row f belongs to image face_image[f]."""
    counts = np.asarray(counts, np.int64).reshape(-1)
    first = np.zeros(counts.shape, np.int64)
    np.cumsum(counts[:-1], out=first[1:])
    return first.astype(np.int32), np.repeat(np.arange(len(counts)), counts).astype(np.int32)


def result_fields(n_images, top_k, n_points, pose, align=None):
    """{name: (shape, dtype name)} of new_results(n_images)."""
    rows = n_images * top_k
    f = {"count": ((n_images,), "int32"), "first": ((n_images,), "int32"), "box": ((rows, 4), "float32"),
         "kps": ((rows, n_points, 2), "float32"), "scores": ((rows, n_points), "float32")}
    if align is not None:
        f.update({"chip": ((rows, align, align, 3), "uint8"), "M": ((rows, 2, 3), "float64")})
    if pose:
        f.update({k: ((rows,) + tail, "float64") for k, tail in POSE_FIELDS})
    return f


class FaceAnaImages:
    def __init__(self, top_k=None, det_input=None, pose=False, max_frames=16, max_faces=64, device="cuda", align=None):
        """top_k: None (Skps.yml's Detect.topk, 5), or 1..1024 faces per image.  det_input: None (Skps.yml's 384x640), or
        the detector input size (h, w) as FaceAna(det_input=...) takes it.  pose: every result dict then also carries
        'pose' as FaceAna(pose=True) returns it, each face with its own image's size for the camera.  align: None, or a
        chip side in 16..512: every result dict then also carries 'chip' (align, align, 3) uint8 and 'M' (2, 3) float64
        as FaceAna(align=align) returns them (FaceLandmark(align=...)'s chip stage).

        run_batch(images)[i] is bit for bit what FaceAna(top_k=top_k, det_input=det_input, pose=pose,
        align=align).run(images[i]) returns on a new or just-reset FaceAna, for images of any size (FaceAna's
        max_frame_hw does not apply).

        max_frames: images per detector forward; max_faces: faces per landmark forward.  A call takes any number of
        images and faces and runs them in chunks of these.  Memory: the detector holds about 39 MB of activations per
        frame of max_frames at 384x640 (0.35 GB at 1152x1920), the landmark net about 47 MB per face of max_faces (3 GB
        at 64).  Each of the two call slots keeps, per image of its largest call, every detector row as a possible kept
        row (rows x 68 bytes: 1.0 MB at 384x640, 9.3 MB at 1152x1920) and top_k selected boxes; per face of its
        largest call, its results (about 1.2 kB, 1.4 kB with pose; with align, align^2 x 3 bytes more on the device and
        as much pinned: 37.6 kB at 112, 786 kB at 512); and, for host images, the pinned staging of the rows and crop
        rectangles it uploads.  With align, one more pinned staging holds the chip rectangles of the largest host call."""
        cfg = get_cfg()['Skps']
        self.top_k = int(top_k if top_k is not None else cfg['Detect']['topk'])
        if not 1 <= self.top_k <= MAX_TOP_K:
            raise ValueError("top_k %d outside 1..%d" % (self.top_k, MAX_TOP_K))
        if det_input is not None:
            det_input = check_detector_input(det_input)
            cfg['Detect']['input_shape'] = [det_input[0], det_input[1], 3]
        self.pose = bool(pose)
        self.align = None if align is None else check_size(align)
        self.detector = FaceDetector(cfg['Detect'], max_frames=max_frames, device=device)
        self.landmark = FaceLandmark(cfg['Keypoints'], max_faces=max_faces, device=device, align=self.align)
        self.max_frames, self.max_faces = self.detector.max_frames, self.landmark.max_faces
        self.device = self.detector.device
        self.n_points = self.landmark.keypoints_num
        self.min_face = float(cfg['Detect']['min_face'])
        # judge_boxs (facer.py:144-189) in numpy's float32: alpha * rect + (1 - alpha) * box, (1 - alpha) in float64 first
        self.iou_thres = float(cfg['Trace']['iou_thres'])
        self.alpha = float(cfg['Trace']['smooth_box'])
        self.one_minus_alpha = 1 - self.alpha
        self.lib = rt.load_library()
        self._slots = None            # device and pinned buffers of the two call slots, made on first use
        self._pending = []            # [(slot, n images, out or None, counts, first, host images to align or None)]
        self._next = 0

    # ------------------------------------------------------------------
    def run_batch(self, images, layout="bgr", rotate=0):
        """FaceAna.run after reset() for every image (blocking): one list of {'box', 'kps', 'scores'[, 'chip', 'M']
        [, 'pose']} per image, [] for an image without a face.  See submit() for what images, layout and rotate may
        be."""
        if self._pending:
            raise RuntimeError("FaceAnaImages: %d calls in flight; collect() them first" % len(self._pending))
        self.submit(images, layout=layout, rotate=rotate)
        return self.collect()

    def new_results(self, n_images):
        """Device result buffers for submit(cuda_images, out=...) of up to n_images images: a dict of CUDA tensors on
        this object's device.  count, first (n,) int32; box (n*top_k, 4), kps (n*top_k, P, 2), scores (n*top_k, P)
        float32; with align also chip (n*top_k, s, s, 3) uint8 and M (n*top_k, 2, 3) float64; with pose also rvec,
        tvec, euler (n*top_k, 3) and reproject (n*top_k, 8, 2) float64.  Faces are packed
        in image order, each image's in FaceAna's order: image i's are rows first[i] .. first[i] + count[i] - 1.  Rows
        past the call's faces are unspecified."""
        rt.require_cuda()
        return new_buffers(result_fields(int(n_images), self.top_k, self.n_points, self.pose, self.align), self.device)

    def submit(self, images, out=None, layout="bgr", rotate=0):
        """Enqueue the analysis of images; at most two calls may be in flight and collect() returns them in submission
        order.  Everything is checked before anything is enqueued.  submit() returns once the call's landmark phase is
        enqueued: the face counts are read back once on the way, so it waits for the call's detector phase.

        images: all HxWx3 uint8 BGR numpy arrays, or all torch.uint8 CUDA tensors (H, W, 3) on this object's device
        with stride(2) == 1, stride(1) == 3 and any row pitch; a mix raises ValueError.  Sizes may differ, as long as
        their letterbox fills the detector input (FaceDetector.submit's rule).  A host image sends only the rows the
        letterbox reads (when fewer than its rows) and the rectangles its crops read; a CUDA image is read where it is.
        Ordering on torch.cuda.current_stream(): CUDA images are read after the work already queued on it, and work
        queued on it after submit() returns runs after they have been read, so the producer may reuse them at once.
        out: None (collect() returns lists of dicts), or, with CUDA images, a dict from new_results(n) with n >= the
        call's images, not used by a call still in flight: the results are written there on the GPU.
        layout: the pixel layout of all CUDA images of the call (device_frames.frame_layout): "bgr" (the default),
        "rgb", "bgra", "rgba" (H, W, 4), "bgr_planar" or "rgb_planar" (3, H, W).  Letterbox, crops and chips read them in
        place, and the results are, bit for bit, those of the same pixels passed as interleaved BGR.  Host images are
        BGR only.
        rotate: the clockwise angle in degrees (0, 90, 180 or 270) by which CUDA images, as stored, must be turned to be
        upright (device_frames.check_rotate), one for the call or one per image (a photo's EXIF orientation, which GPU
        JPEG decoders do not apply).  They are read in place, and every result, pose included, is in the upright
        image's pixels, bit for bit that of the upright image passed as a contiguous tensor.  Host images take 0.

        With align, CUDA images are warped into chips right after the landmarks, with no host synchronisation.  Host
        images are warped at collect(): M comes back with the other results, and only the rectangle of an image each
        chip reads is uploaded then.  That is one more read-back and one more upload per call, and the host images
        must stay unchanged until collect() returns."""
        if len(self._pending) == 2:
            raise RuntimeError("FaceAnaImages: two calls already in flight; call collect() first")
        fd, fl = self.detector, self.landmark
        call = check_frames(images, self.device, layout, rotate)
        layout = fd._layout(call)
        n = len(call.frames)
        if out is not None:
            if not call.cuda:
                raise ValueError("out= keeps results on the GPU and takes CUDA images")
            check_out(out, result_fields(n, self.top_k, self.n_points, self.pose, self.align), self.device,
                      [p[2] for p in self._pending])
        if n == 0:
            self._pending.append((None, 0, None, None, None, None))
            return
        torch = rt.require_cuda()
        if self._slots is None:
            self._slots = [self._new_slot() for _ in range(2)]
        slot = self._next
        st = self._slots[slot]
        K, P, lib = self.top_k, self.n_points, self.lib
        ds, ls = fd.model.stream, fl.model.stream

        # 1. detector: every kept row of every image stays on the device
        cpad = pad16(n)
        if st["det"] is None or st["det"]["count"].shape[0] < n:
            st["done"].synchronize()                  # the slot's last call has finished with what is replaced
            st["det"] = fd.new_results(max(n, 0 if st["det"] is None else 2 * st["det"]["count"].shape[0]))
        need = cpad + 4 * n * K
        if st["sel"] is None or st["sel"].shape[0] < need:
            st["done"].synchronize()
            st["sel"] = grow(st["sel"], need, lambda k: torch.empty((k,), dtype=torch.float32, device=self.device))
            st["hsel"] = grow(st["hsel"], need, lambda k: torch.empty((k,), dtype=torch.float32).pin_memory())
        # The detector starts after the previous call's landmark phase, so the two engines never run at the same time:
        # landmarks computed while the other engine ran on another stream have been seen to vary from run to run.  The
        # next call's host staging still overlaps the GPU work.  This also orders the slot's last reads of its boxes.
        ds.wait_event(self._slots[slot ^ 1]["done"])
        ds.wait_event(st["done"])
        fd._enqueue(call, layout, st["det"], detect=True)
        # 2. face selection, all images in one launch; 3. the call's one read-back: counts and selected boxes
        sel = st["sel"]
        with torch.cuda.device(self.device):          # the kernels launch on the current device
            rt.check(lib.skps_select_faces_batch(st["det"]["rows"].data_ptr(), st["det"]["count"].data_ptr(), fd._rows,
                                                 n, self.min_face, K, sel.data_ptr() + 4 * cpad, sel.data_ptr(),
                                                 ds.cuda_stream))
        with torch.cuda.stream(ds):
            st["hsel"][:need].copy_(sel[:need], non_blocking=True)
        st["selected"].record(ds)
        st["selected"].synchronize()
        hsel = st["hsel"].numpy()
        counts = hsel[:n].view(np.int32).copy()
        boxes = hsel[cpad:need].reshape(n, K, 4)
        first, face_image = pack_faces(counts)
        F = int(counts.sum())

        # 4. landmarks on exactly the faces found, packed in image order
        if out is None:
            self._grow_faces(st, max(F, 1))
            res = {k: st[k] for k in self._face_fields(0)}
        else:
            res = out
        fl._enqueue(call, *fl._check_boxes(call, [boxes[i, :k] for i, k in enumerate(counts.tolist())]),
                    {k: res[k] for k in fl._fields(0)})
        # face -> image map and each face's image size; with out=, first and count too: one upload
        m = 2 * n + 3 * F
        if st["hmap"] is None or st["hmap"].shape[0] < m:
            st["done"].synchronize()
            st["hmap"] = grow(st["hmap"], m, lambda k: torch.empty((k,), dtype=torch.int32).pin_memory())
            st["map"] = grow(st["map"], m, lambda k: torch.empty((k,), dtype=torch.int32, device=self.device))
        st["staged"].synchronize()                    # the slot's last upload has left the pinned map
        hmap = st["hmap"].numpy()
        hmap[:n], hmap[n:2 * n], hmap[2 * n:2 * n + F] = first, counts, face_image
        hw = np.array(call.upright, np.int32).reshape(-1, 2)
        hmap[2 * n + F:m].reshape(F, 2)[:] = hw[face_image]
        dmap = st["map"]
        with torch.cuda.stream(ls):
            dmap[:m].copy_(st["hmap"][:m], non_blocking=True)
            st["staged"].record(ls)
            if out is not None:
                out["first"][:n].copy_(dmap[:n])
                out["count"][:n].copy_(dmap[n:2 * n])
        # 5. the returned box; 6. head pose
        face_ptr, hw_ptr = dmap.data_ptr() + 4 * 2 * n, dmap.data_ptr() + 4 * (2 * n + F)
        with torch.cuda.device(self.device):
            rt.check(lib.skps_landmark_boxes(res["kps"].data_ptr(), P, face_ptr, F, sel.data_ptr() + 4 * cpad,
                                             sel.data_ptr(), K, self.iou_thres, self.alpha, self.one_minus_alpha,
                                             res["box"].data_ptr(), ls.cuda_stream))
            if self.pose:
                rt.check(lib.skps_head_pose_faces(res["kps"].data_ptr(), F, P, hw_ptr, res["rvec"].data_ptr(),
                                                  res["tvec"].data_ptr(), res["euler"].data_ptr(),
                                                  res["reproject"].data_ptr(), ls.cuda_stream))
        # 7. results: back to pinned host memory, or left in out
        if out is None and F:
            with torch.cuda.stream(ls):
                for k, t in res.items():
                    if k != "chip" or call.cuda:      # host images are warped at collect()
                        st["h" + k][:F].copy_(t[:F], non_blocking=True)
        st["done"].record(ls)
        align_host = self.align is not None and not call.cuda
        self._pending.append((slot, n, out, counts, first, call if align_host else None))
        self._next ^= 1

    def collect(self):
        """Results of the oldest call in flight: one list of {'box', 'kps', 'scores'[, 'pose']} per image, as FaceAna.run
        returns them; for a call submitted with out=, the out dict, with no host synchronisation:
        torch.cuda.current_stream() is made to wait for the call, so work queued on it afterwards sees the results."""
        if not self._pending:
            raise RuntimeError("FaceAnaImages: nothing submitted")
        slot, n, out, counts, first, host_call = self._pending.pop(0)
        if n == 0:
            return []
        st = self._slots[slot]
        if out is not None:
            import torch
            torch.cuda.current_stream(self.device).wait_event(st["done"])
            return out
        st["done"].synchronize()
        F = int(counts.sum())
        if host_call is not None and F:
            fl = self.landmark
            fl.host_chips.warp(fl.lib, fl.model.stream, host_call, counts.tolist(), st["hM"].numpy()[:F], st["chip"],
                               st["hchip"])
        host = {k: st["h" + k].numpy()[:F] for k in self._face_fields(0)}
        res = []
        for o, k in zip(first.tolist(), counts.tolist()):
            part = {name: a[o:o + k].copy() for name, a in host.items()}
            faces = [{'box': part['box'][j], 'kps': part['kps'][j], 'scores': part['scores'][j]} for j in range(k)]
            if self.align is not None:
                for j, r in enumerate(faces):
                    r['chip'], r['M'] = part['chip'][j], part['M'][j]
            if self.pose:
                for j, r in enumerate(faces):
                    r['pose'] = {name: part[name][j] for name, _ in POSE_FIELDS}
            res.append(faces)
        return res

    # ------------------------------------------------------------------
    def _new_slot(self):
        import torch
        ev = {name: torch.cuda.Event() for name in ("selected", "staged", "done")}
        return dict(det=None, sel=None, hsel=None, map=None, hmap=None, faces=0, **ev)

    def _face_fields(self, rows):
        """The per-face fields of result_fields, for `rows` faces."""
        f = result_fields(rows, 1, self.n_points, self.pose, self.align)
        del f["count"], f["first"]
        return f

    def _grow_faces(self, st, F):
        """The slot's device results and their pinned copies, for at least F faces."""
        if st["faces"] >= F:
            return
        st["done"].synchronize()
        rows = max(F, 2 * st["faces"], 1)
        fields = self._face_fields(rows)
        st.update(new_buffers(fields, self.device))
        st.update({"h" + k: t.pin_memory() for k, t in new_buffers(fields, "cpu").items()})
        st["faces"] = rows
