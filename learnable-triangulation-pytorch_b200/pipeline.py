"""Host-side batch contract on either side of the forward path, GPU-first (SURVEY.md 8(f) row 3).

Mirrors `/root/reference/mvn/datasets/utils.py`: `make_collate_fn` (:6-39), `worker_init_fn`
(:42-43) and `prepare_batch` (:45-65) with the same names, arguments and return values, but:

  * the collate writes the items straight into ONE (optionally pinned) staging array instead of
    two nested `np.stack` passes plus a strided `swapaxes` view;
  * `prepare_batch` uploads the raw HWC buffer once and does transpose + cast (+ ImageNet
    normalisation of uint8 crops through a 256-entry table, img.py:102-110) in
    `lt_images_hwc_to_nchw_fwd` on the GPU -- the reference transposes/casts every view on the CPU
    (`image_batch_to_torch`, img.py:96-99) and uploads it view by view from pageable memory;
  * projection matrices come from one vectorised float64 product (`multiview.stack_projections`)
    instead of B*V `torch.from_numpy(camera.projection)` calls.

`InferenceStream` is the serving loop built on top: host->device copies of batch i+1 run on a copy
stream while batch i computes (CUDA-graph replay), results return through pinned memory.
"""
import collections

import numpy as np
import torch

from . import capi, multiview
from .op import _resolve_backend

IMAGENET_MEAN = np.array([0.485, 0.456, 0.406])    # img.py:7
IMAGENET_STD = np.array([0.229, 0.224, 0.225])


def normalization_table(mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """float32 [C][256]: table[c][u] = float32((u / 255.0 - mean[c]) / std[c]), evaluated in float64 exactly as
    `normalize_image` (img.py:102-110) does for a uint8 image, so a lookup equals normalise-then-`.float()`."""
    u = np.arange(256, dtype=np.float64)[None, :]
    mean = np.asarray(mean, dtype=np.float64)[:, None]
    std = np.asarray(std, dtype=np.float64)[:, None]
    return ((u / 255.0 - mean) / std).astype(np.float32)


def pinned_empty(shape, dtype):
    """numpy array backed by page-locked memory (so `.to(device, non_blocking=True)` is a true async DMA)."""
    tdtype = {np.dtype(np.uint8): torch.uint8, np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64}[np.dtype(dtype)]
    pin = torch.cuda.is_available()
    return torch.empty(tuple(shape), dtype=tdtype, pin_memory=pin).numpy()


def make_collate_fn(randomize_n_views=True, min_n_views=10, max_n_views=31, pinned=False):
    """Same contract as reference datasets/utils.py:6-39.  `batch['images']` is a contiguous (B, n_views, H, W, C)
    array (the reference returns a strided view of a (n_views, B, ...) stack with the same values); with
    `pinned=True` it lives in page-locked memory.  Note a pinned array must stay in the process that uploads it
    (use it with `num_workers=0` or a thread-based loader)."""

    def collate_fn(items):
        items = [item for item in items if item is not None]
        if len(items) == 0:
            print("All items in batch are None")
            return None
        total_n_views = min(len(item["images"]) for item in items)
        if randomize_n_views:
            n_views = np.random.randint(min_n_views, min(total_n_views, max_n_views) + 1)
            indexes = np.random.choice(np.arange(total_n_views), size=n_views, replace=False)
        else:
            indexes = np.arange(total_n_views)

        first = np.asarray(items[0]["images"][int(indexes[0])])
        shape = (len(items), len(indexes)) + first.shape
        images = pinned_empty(shape, first.dtype) if pinned else np.empty(shape, dtype=first.dtype)
        for b, item in enumerate(items):
            for j, i in enumerate(indexes):
                images[b, j] = item["images"][int(i)]

        batch = dict()
        batch["images"] = images
        batch["detections"] = np.array([[item["detections"][int(i)] for i in indexes] for item in items])
        batch["cameras"] = [[item["cameras"][int(i)] for item in items] for i in indexes]     # [view][batch]
        batch["keypoints_3d"] = [item["keypoints_3d"] for item in items]
        batch["indexes"] = [item["indexes"] for item in items]
        try:
            batch["pred_keypoints_3d"] = np.array([item["pred_keypoints_3d"] for item in items])
        except Exception:
            pass
        return batch

    return collate_fn


def worker_init_fn(worker_id):
    np.random.seed(np.random.get_state()[1][0] + worker_id)


class HostStager:
    """Reusable page-locked staging buffers keyed by (shape, dtype): pageable batches are copied in once and
    uploaded with an asynchronous DMA; arrays that already live in pinned memory are uploaded as they are."""

    def __init__(self, depth=2):
        self.depth = depth
        self._pools = collections.defaultdict(list)
        self._next = collections.defaultdict(int)

    def stage(self, array):
        t = torch.from_numpy(array)
        if t.is_pinned() or not torch.cuda.is_available():
            return t
        key = (tuple(array.shape), array.dtype.str)
        pool = self._pools[key]
        if len(pool) < self.depth:
            pool.append(torch.empty(tuple(array.shape), dtype=t.dtype, pin_memory=True))
        buf = pool[self._next[key] % len(pool)]
        self._next[key] += 1
        buf.copy_(t)
        return buf


_default_stager = HostStager()
_lut_cache = {}


def _device_lut(device):
    key = (device.type, device.index)
    if key not in _lut_cache:
        _lut_cache[key] = torch.from_numpy(normalization_table()).to(device)
    return _lut_cache[key]


def images_to_device(images, device, normalize_u8=False, backend=None, stager=None):
    """(B, V, H, W, C) host array (uint8 / float32 / float64, as collated) -> (B, V, C, H, W) float32 on `device`.

    Equals `torch.stack([image_batch_to_torch(x).to(device) for x in images])` (datasets/utils.py:47-52); with
    `normalize_u8=True` uint8 input is additionally mapped through `normalize_image` (img.py:102-110) bit-exactly.
    """
    images = np.asarray(images)
    if images.dtype not in (np.uint8, np.float32, np.float64):
        images = images.astype(np.float32)
    images = np.ascontiguousarray(images)
    B, V, H, W, C = images.shape
    device = torch.device(device)
    probe = torch.empty(0, device=device)
    if _resolve_backend(backend, probe) == "torch":
        t = torch.from_numpy(images)
        if normalize_u8 and images.dtype == np.uint8:
            lut = torch.from_numpy(normalization_table())                        # [C][256]
            t = lut[torch.arange(C).view(1, 1, 1, 1, C), t.long()]
        return t.permute(0, 1, 4, 2, 3).float().contiguous().to(device)
    staged = (stager or _default_stager).stage(images)
    raw = staged.to(device, non_blocking=True)
    out = torch.empty((B, V, C, H, W), dtype=torch.float32, device=device)
    lut = _device_lut(device) if (normalize_u8 and images.dtype == np.uint8) else None
    capi.images_hwc_to_nchw(raw, lut, out, B * V, C, H, W)
    return out


def prepare_batch(batch, device, config=None, is_train=True, normalize_u8=False, backend=None, stager=None):
    """Drop-in for reference datasets/utils.py:45-65: returns
    (images (B,V,3,H,W), keypoints_3d_gt (B,J,3), keypoints_3d_validity_gt (B,J,1), proj_matricies (B,V,3,4)),
    all float32 on `device`.  `config` and `is_train` are accepted and unused, as in the reference."""
    device = torch.device(device)
    images_batch = images_to_device(batch["images"], device, normalize_u8=normalize_u8, backend=backend, stager=stager)
    kp = np.stack(batch["keypoints_3d"], axis=0)
    keypoints_3d_batch_gt = torch.from_numpy(np.ascontiguousarray(kp[:, :, :3], dtype=np.float32)).to(device)
    keypoints_3d_validity_batch_gt = torch.from_numpy(np.ascontiguousarray(kp[:, :, 3:], dtype=np.float32)).to(device)
    proj_matricies_batch = torch.from_numpy(multiview.stack_projections(batch["cameras"])).to(device)
    return images_batch, keypoints_3d_batch_gt, keypoints_3d_validity_batch_gt, proj_matricies_batch


class InferenceStream:
    """Pipelined serving loop over host batches.

        stream = InferenceStream(model)                    # model: VolumetricTriangulationNet on a CUDA device, eval
        for keypoints in stream.run(batches):              # batches: iterable of collated batch dicts
            ...                                            # keypoints: (B, J, 3) float32 numpy array

    Per batch, inside the loop: pageable->pinned staging (skipped for pinned collates), host->device DMA of the raw HWC
    images on a copy stream, layout/normalisation kernel, the model forward (CUDA-graph replay) and an asynchronous
    device->host copy of the keypoints into pinned memory.  The upload of batch i+1 overlaps the forward of batch i;
    results are yielded in order, one batch behind the submission front.
    """

    def __init__(self, model, normalize_u8=False, depth=2):
        self.model = model
        self.device = next(model.parameters()).device
        if self.device.type != "cuda":
            raise RuntimeError("InferenceStream drives the native CUDA path; the model must live on a CUDA device")
        self.normalize_u8 = normalize_u8
        self.depth = depth
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self.stager = HostStager(depth=depth + 1)
        self._raw = {}       # (slot, shape, dtype) -> device buffer for the raw upload
        self._out = {}       # slot -> pinned result buffer
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    def _upload(self, slot, images, consumed_event):
        images = np.ascontiguousarray(images)
        staged = self.stager.stage(images)
        key = (slot, tuple(images.shape), images.dtype.str)
        if key not in self._raw:
            self._raw[key] = torch.empty(tuple(images.shape), dtype=staged.dtype, device=self.device)
        raw = self._raw[key]
        with torch.cuda.stream(self.copy_stream):
            if consumed_event is not None:
                self.copy_stream.wait_event(consumed_event)      # the kernel that last read this slot has finished
            raw.copy_(staged, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(self.copy_stream)
        self.h2d_bytes += images.nbytes
        return raw, ready

    def _launch(self, slot, raw, ready, batch):
        main = torch.cuda.current_stream(self.device)
        main.wait_event(ready)
        B, V, H, W, C = raw.shape
        images = torch.empty((B, V, C, H, W), dtype=torch.float32, device=self.device)
        lut = _device_lut(self.device) if (self.normalize_u8 and raw.dtype == torch.uint8) else None
        capi.images_hwc_to_nchw(raw, lut, images, B * V, C, H, W)
        consumed = torch.cuda.Event()
        consumed.record(main)
        keypoints = self.model(images, None, batch)[0]
        out = self._out.get((slot, tuple(keypoints.shape)))
        if out is None:
            out = torch.empty(tuple(keypoints.shape), dtype=torch.float32, pin_memory=True)
            self._out[(slot, tuple(keypoints.shape))] = out
        out.copy_(keypoints, non_blocking=True)
        done = torch.cuda.Event()
        done.record(main)
        self.d2h_bytes += out.numel() * 4
        return out, done, consumed

    def run(self, batches):
        pending = collections.deque()       # (pinned result, done event)
        consumed = [None] * self.depth
        it = iter(batches)
        nxt = next(it, None)
        i = 0
        staged_next = None
        if nxt is not None:
            staged_next = self._upload(0, nxt["images"], None)
        with torch.no_grad():
            while nxt is not None:
                cur, (raw, ready) = nxt, staged_next
                slot = i % self.depth
                nxt = next(it, None)
                if nxt is not None:                                   # start the next upload before launching this forward
                    nslot = (i + 1) % self.depth
                    staged_next = self._upload(nslot, nxt["images"], consumed[nslot])
                out, done, cons = self._launch(slot, raw, ready, cur)
                consumed[slot] = cons
                pending.append((out, done))
                if len(pending) >= self.depth:                        # result buffers are per slot: drain before reuse
                    o, d = pending.popleft()
                    d.synchronize()
                    yield o.numpy().copy()
                i += 1
            while pending:
                o, d = pending.popleft()
                d.synchronize()
                yield o.numpy().copy()
