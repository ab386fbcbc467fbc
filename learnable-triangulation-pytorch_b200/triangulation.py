"""Drop-in `VolumetricTriangulationNet` (reference mvn/models/triangulation.py:203-355).

Same constructor (`config`, `device`), same `forward(images, proj_matricies, batch)` 7-tuple, same
attribute names (`backbone`, `process_features`, `volume_net`) and `state_dict()` keys, same
config side effects (triangulation.py:228-231) -- so the reference `train.py` can construct, load,
wrap in DDP and call it unchanged.

backend="native" (default; eval/no-grad on a CUDA device): host geometry is vectorised numpy
(float64, cast last, like the reference) and everything on the device runs in the hand-written
sm_90a kernels through engine.NativeEngine.  backend="torch": autograd-capable torch ops
(training, CPU plumbing).  Nothing switches backend silently.
"""
import collections.abc
import os
import random

import numpy as np
import torch
from torch import nn

from . import autograd_ops, capi, layers, multiview, op, pose_resnet, torch_ops, volumetric
from .train_graph import TrainGraphs
from .v2v import V2VModel


def backbone_map_size(size):
    """Spatial size of the backbone's heat-map / feature output for an input side `size` (pose_resnet.py:293-313):
    7x7 s2 p3 stem, 3x3 s2 p1 max-pool, three 3x3 s2 p1 stages, three k4 s2 p1 transposed convs.  This is the same
    arithmetic the engine's launch plan follows, so the intrinsics are rescaled by the size the kernels really produce
    (the reference reads it off `heatmaps.shape`, triangulation.py:264-265)."""
    s = (size + 6 - 7) // 2 + 1
    s = (s + 2 - 3) // 2 + 1
    for _ in range(3):
        s = (s + 2 - 3) // 2 + 1
    return s * 8


def _base_points(batch, batch_size, kind, use_gt_pelvis):
    """Pelvis (mpii: joint 6) or hip midpoint (coco) per sample, float64 (triangulation.py:286-296)."""
    pts = np.empty((batch_size, 3), dtype=np.float64)
    for b in range(batch_size):
        kp = batch["keypoints_3d"][b] if use_gt_pelvis else batch["pred_keypoints_3d"][b]
        if kind == "coco":
            pts[b] = (kp[11, :3] + kp[12, :3]) / 2
        elif kind == "mpii":
            pts[b] = kp[6, :3]
        else:
            raise KeyError("unknown skeleton kind {!r}".format(kind))
    return pts


def _place_cuboids(base, sides):
    """Cuboid corner base - sides / 2 (B, 3) float64 and the per-sample volumetric.Cuboid3D (triangulation.py:298-303)."""
    position = base - sides / 2
    return position, [volumetric.Cuboid3D(position[b], sides) for b in range(base.shape[0])]


_NO_V2V = object()      # the v2v_backend of a model without a V2V net (None stays an unknown v2v_backend)


def _check_backends(backend, conv_mode, backbone_backend, norm_backend, v2v_backend=_NO_V2V, head_backend="torch", eval_backend=None):
    """ValueError unless the training switches are known values in a supported combination.

    eval_backend="native": an eval-mode forward without gradients of a backend="torch" / "hybrid" model runs the native engine, as
    a backend="native" model with the same weights does (packed filters, folded BatchNorm, CUDA graphs).  Every other forward is
    unchanged; with backend="native" it changes nothing.  None (the default) never uses the engine.

    v2v_backend="native" / backbone_backend="native": every Conv3d / ConvTranspose3d of volume_net / every Conv2d / ConvTranspose2d
    of the backbone, its confidence heads and `process_features` runs forward, data gradient and weight gradient on the native
    tensor-core kernels.  Both need backend="hybrid" and conv_mode="tc".
    norm_backend="native": every BatchNorm2d / BatchNorm3d of the backbone, its confidence heads and the V2V net, fused with the ReLU
    after it and the residual add of a residual unit, trains on the native kernels.  The kernels read the channels-last maps the
    native convolutions produce, so it needs backend="hybrid" and every conv switch of the model "native".
    head_backend="native": the confidence heads' tail (second max pool, ReLU, global mean, the three Linear layers and the sigmoid) and
    the normalisation of the confidences over the views train on the native kernels, forward and backward, without cuBLAS.  It needs
    backend="hybrid" and composes with every other switch; a model without confidence heads runs unchanged."""
    convs = [("backbone_backend", backbone_backend)] + ([] if v2v_backend is _NO_V2V else [("v2v_backend", v2v_backend)])
    for name, value in reversed(convs):     # the V2V switch first
        if value not in ("torch", "native"):
            raise ValueError("unknown {} {!r}".format(name, value))
        if value == "native" and (backend != "hybrid" or conv_mode != "tc"):
            raise ValueError("%s='native' needs backend='hybrid' and conv_mode='tc' (got %r, %r)" % (name, backend, conv_mode))
    if norm_backend not in ("torch", "native"):
        raise ValueError("unknown norm_backend {!r}".format(norm_backend))
    if norm_backend == "native" and (backend != "hybrid" or any(value != "native" for _, value in convs)):
        raise ValueError("norm_backend='native' needs backend='hybrid' and %s (got backend=%r, %s)"
                         % (" and ".join("%s='native'" % name for name, _ in convs), backend, ", ".join("%s=%r" % c for c in convs)))
    if head_backend not in ("torch", "native"):
        raise ValueError("unknown head_backend {!r}".format(head_backend))
    if head_backend == "native" and backend != "hybrid":
        raise ValueError("head_backend='native' needs backend='hybrid' (got %r)" % (backend,))
    if eval_backend not in (None, "native"):
        raise ValueError("unknown eval_backend {!r} (None or 'native')".format(eval_backend))


def _hooks(backbone_backend, norm_backend, v2v_backend="torch"):
    """(backbone conv, V2V conv, norm) hooks of checked switches: the torch formulas in layers.py for "torch", autograd_ops'
    native training functions for "native"."""
    return (autograd_ops.backbone_conv if backbone_backend == "native" else layers.torch_conv,
            autograd_ops.v2v_conv if v2v_backend == "native" else layers.torch_conv,
            autograd_ops.batch_norm if norm_backend == "native" else layers.torch_norm)


def _head_tail(head_backend):
    """The confidence heads' `tail` hook of a checked head_backend: None (the torch modules) or autograd_ops.conf_head_tail."""
    return autograd_ops.conf_head_tail if head_backend == "native" else None


def _upload(device, *arrays, dtype=torch.float32):
    """`dtype` (float32 by default) tensors on `device` of host arrays (float64 cast last): on CUDA through one page-locked buffer
    and one asynchronous copy, so the host part of a forward does not wait for the device."""
    flat = [torch.from_numpy(np.ascontiguousarray(a)).to(dtype).reshape(-1) for a in arrays]
    host = torch.cat(flat)
    if device.type == "cuda":
        host = host.pin_memory().to(device, non_blocking=True)
    return tuple(t.view(a.shape) for t, a in zip(host.split([f.numel() for f in flat]), arrays))


def _check_train_graph(train_graph, backend):
    if train_graph and backend != "hybrid":
        raise ValueError("train_graph=True needs backend='hybrid' (got %r)" % (backend,))


class _EngineOwner(nn.Module):
    """Keeps the native engine's packed filters / CUDA graphs and the training graphs (train_graph.TrainGraphs, TrainStep) in step with the
    module's tensors: `.to()/.cuda()/.float()` (`_apply`) and `load_state_dict` invalidate them explicitly (tensor versions alone
    miss `p.data` updates)."""

    def _invalidate_engine(self):
        eng = self.__dict__.get("_engine")
        if eng is not None:
            eng.invalidate()
        graphs = self.__dict__.get("_train_graphs")
        if graphs is not None:
            graphs.invalidate()
        for step in self.__dict__.get("_train_steps", ()):        # train_graph.TrainStep graphs of this model
            step.invalidate()

    def _run_device(self, fn, inputs):
        """fn(*inputs): the device part of a torch / hybrid forward, replayed from CUDA graphs with train_graph=True in a training
        forward.  A train-mode forward invalidates the native engine (_invalidate_native_eval)."""
        if self.training:
            self._invalidate_native_eval()
        if self._train_graphs is not None and self.training and torch.is_grad_enabled():
            return self._train_graphs.run(self, fn, inputs, self.clone_outputs)
        return fn(*inputs)

    def _invalidate_native_eval(self):
        """Drop the native engine's packed filters and graphs, keeping the training graphs: training changes weights and BatchNorm
        statistics where NativeEngine._param_version cannot see it (TrainStep's captured Adam, replayed BatchNorm updates, the native
        BatchNorm's pointer writes).  Called by every train-mode forward and every TrainStep call, so the next eval_backend="native"
        forward re-packs and re-captures, and the eval graphs and packs are not held during training."""
        eng = self.__dict__.get("_engine")
        if eng is not None:
            eng.invalidate()

    def _native_eval(self):
        """Whether this forward of a torch / hybrid model runs on the native engine: eval_backend="native", eval mode, no grad."""
        return self.eval_backend == "native" and not self.training and not torch.is_grad_enabled()

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self._invalidate_engine()
        return out

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        self._invalidate_engine()
        return out


class VolumetricTriangulationNet(_EngineOwner):
    def __init__(self, config, device="cuda:0", backend=None, conv_mode=None, use_cuda_graph=True, v2v_backend="torch",
                 backbone_backend="torch", norm_backend="torch", train_graph=False, head_backend="torch", eval_backend=None):
        super().__init__()
        m = config.model
        self.num_joints = m.backbone.num_joints
        self.volume_aggregation_method = m.volume_aggregation_method
        self.volume_softmax = m.volume_softmax
        self.volume_multiplier = m.volume_multiplier
        self.volume_size = m.volume_size
        self.cuboid_side = m.cuboid_side
        self.kind = m.kind
        self.use_gt_pelvis = m.use_gt_pelvis
        self.heatmap_softmax = m.heatmap_softmax
        self.heatmap_multiplier = m.heatmap_multiplier
        self.transfer_cmu_to_human36m = m.transfer_cmu_to_human36m if hasattr(m, "transfer_cmu_to_human36m") else False

        # the reference mutates the caller's config here (triangulation.py:228-231); so do we
        m.backbone.alg_confidences = False
        m.backbone.vol_confidences = False
        if self.volume_aggregation_method.startswith("conf"):
            m.backbone.vol_confidences = True

        self.backbone = pose_resnet.get_pose_net(m.backbone, device=device)
        for p in self.backbone.final_layer.parameters():
            p.requires_grad = False
        self.process_features = nn.Sequential(nn.Conv2d(256, 32, 1))
        self.volume_net = V2VModel(32, self.num_joints)

        self.backend = backend or os.environ.get("LT_B200_BACKEND", "native")
        self.conv_mode = conv_mode or os.environ.get("LT_B200_CONV", "tc")
        _check_backends(self.backend, self.conv_mode, backbone_backend, norm_backend, v2v_backend, head_backend, eval_backend)
        _check_train_graph(train_graph, self.backend)
        self.v2v_backend = v2v_backend
        self.head_backend = head_backend
        self.eval_backend = eval_backend
        self.backbone_backend = backbone_backend
        self.norm_backend = norm_backend
        self.use_cuda_graph = use_cuda_graph
        self.clone_outputs = True
        self._engine = None
        self._train_graphs = TrainGraphs() if train_graph else None

    # ---------------------------------------------------------------- host-side geometry
    def _host_geometry(self, batch, batch_size, image_shape, heatmap_shape):
        base = _base_points(batch, batch_size, self.kind, self.use_gt_pelvis)                 # (B, 3) f64
        proj, sides, step, rots = self._pelvis_free_geometry(batch, batch_size, image_shape, heatmap_shape)
        position, cuboids = _place_cuboids(base, sides)
        return proj, base, position, step, rots, cuboids

    def _pelvis_free_geometry(self, batch, batch_size, image_shape, heatmap_shape):
        """The host geometry that does not depend on the pelvis: heat-map-space projections (B, V, 3, 4) float32, the cuboid sides
        (3,) and voxel step (3,) float64, rotations (B, 3, 3) float64 (a random angle per sample in training)."""
        proj = multiview.stack_projections(batch["cameras"], image_shape, heatmap_shape)
        sides = np.array([self.cuboid_side] * 3, dtype=np.float64)
        axis = [0, 1, 0] if self.kind == "coco" else [0, 0, 1]
        rots = np.empty((batch_size, 3, 3), dtype=np.float64)
        for b in range(batch_size):
            theta = np.random.uniform(0.0, 2 * np.pi) if self.training else 0.0   # triangulation.py:318-321
            rots[b] = volumetric.get_rotation_matrix(axis, theta)
        step = sides / (self.volume_size - 1)
        return proj, sides, step, rots

    def engine(self):
        if self._engine is None:
            from .engine import NativeEngine
            self._engine = NativeEngine(self, mode=self.conv_mode, use_graph=self.use_cuda_graph)
        return self._engine

    # ---------------------------------------------------------------- forward
    def forward(self, images, proj_matricies, batch):
        if self.backend in ("torch", "hybrid") and not self._native_eval():
            # "hybrid": torch/cuDNN convolutions with the native custom ops (forward + backward kernels) in the autograd graph
            return self._forward_torch(images, batch)
        if self.backend not in ("native", "torch", "hybrid"):
            raise ValueError("unknown backend {!r}".format(self.backend))
        return self._forward_native(images, batch)

    def _forward_native(self, images, batch):
        """The native engine's forward: backend="native", and the eval forwards of eval_backend="native"."""
        if not images.is_cuda:
            raise RuntimeError("lt_b200 native backend needs CUDA tensors (got %s); construct the model with "
                               "backend='torch' for the CPU/autograd path" % images.device)
        if self.training or torch.is_grad_enabled():
            raise RuntimeError("lt_b200 native backend is inference-only: call model.eval() under torch.no_grad(), "
                               "or construct the model with backend='torch' (LT_B200_BACKEND=torch) for training")
        B, V = images.shape[:2]
        H, W = images.shape[3:]
        if H % 2 or W % 2:
            raise ValueError("lt_b200 native backend needs even image sides (space-to-depth stem), got %dx%d" % (H, W))
        hm_shape = (backbone_map_size(H), backbone_map_size(W))   # == H // 4 only when H is a multiple of 32
        proj, base, position, step, rots, cuboids = self._host_geometry(batch, B, (H, W), hm_shape)
        dev = images.device
        with torch.cuda.device(dev):      # launches go to the model's device, whatever the caller's current device is
            # one page-locked upload: a pageable copy would wait for the host, and a replayed forward synchronises nowhere
            geometry = _upload(dev, proj, position, base, step, rots.reshape(B, 9))
            outs = self.engine().forward(images.float().contiguous(), *geometry)
            base_points = geometry[2]
        if self.clone_outputs and self.use_cuda_graph:
            outs = tuple(o.clone() for o in outs)
        kp, features, volumes, coord = outs[:4]
        if tuple(features.shape[3:]) != hm_shape:
            raise RuntimeError("feature map %s differs from the heat-map size %s used for the projection matrices"
                               % (tuple(features.shape[3:]), hm_shape))
        vol_conf = outs[4] if len(outs) > 4 else None
        return kp, features, volumes, vol_conf, cuboids, coord, base_points

    def _forward_torch(self, images, batch):
        """backend "torch" / "hybrid": the host part (geometry with the heat-map size of backbone_map_size, its upload), then
        _device_forward, from CUDA graphs with train_graph=True."""
        if self.backend == "hybrid" and not images.is_cuda:
            raise RuntimeError("lt_b200 hybrid backend needs CUDA tensors (native custom ops); use backend='torch' on CPU")
        B = images.shape[0]
        H, W = images.shape[3:]
        hm_shape = (backbone_map_size(H), backbone_map_size(W))
        proj, base, position, step, rots, cuboids = self._host_geometry(batch, B, (H, W), hm_shape)
        geometry = _upload(images.device, proj, position, base, step, rots)
        kp, features, volumes, vol_conf, coord = self._run_device(self._device_forward, (images,) + geometry)
        return kp, features, volumes, vol_conf, cuboids, coord, geometry[2]

    def _device_forward(self, images, proj_t, pos_t, cen_t, step_t, rot_t):
        """Everything the torch / hybrid forward runs on the device: (images, projections (B, V, 3, 4), cuboid position (B, 3), base
        point (B, 3), voxel step (3,), rotations (B, 3, 3)) -> (kp, features, volumes, vol_conf, coord)."""
        dev = images.device
        B, V = images.shape[:2]
        flat = images.reshape(-1, *images.shape[2:])
        conv, v2v_conv, norm = _hooks(self.backbone_backend, self.norm_backend, self.v2v_backend)
        heatmaps, features, _, vol_conf = self.backbone(flat, conv, norm, _head_tail(self.head_backend))
        hm_shape = (backbone_map_size(images.shape[3]), backbone_map_size(images.shape[4]))
        if tuple(heatmaps.shape[2:]) != hm_shape:
            raise RuntimeError("heat-map size %s differs from the size %s used for the projection matrices"
                               % (tuple(heatmaps.shape[2:]), hm_shape))
        if vol_conf is not None:
            vol_conf = vol_conf.view(B, V, *vol_conf.shape[1:])
            if self.volume_aggregation_method == "conf_norm":
                if self.head_backend == "native":
                    vol_conf = autograd_ops.view_normalize(vol_conf, 0.0)
                else:
                    vol_conf = vol_conf / vol_conf.sum(dim=1, keepdim=True)
        n = self.volume_size
        idx = torch.arange(n, device=dev, dtype=torch.float)
        grid = torch.stack(torch.meshgrid(idx, idx, idx, indexing="ij"), dim=-1)              # (n, n, n, 3)
        coord = pos_t.view(B, 1, 1, 1, 3) + step_t * grid.unsqueeze(0)
        coord = coord - cen_t.view(B, 1, 1, 1, 3)
        coord = torch.einsum("bij,bxyzj->bxyzi", rot_t, coord) + cen_t.view(B, 1, 1, 1, 3)
        if self.transfer_cmu_to_human36m:
            coord = coord.permute(0, 1, 3, 2, 4).flip(2)
        features = layers.run(self.process_features, features, conv, norm)
        features = features.view(B, V, *features.shape[1:])
        ops = autograd_ops if self.backend == "hybrid" else torch_ops
        volumes = ops.unproject_heatmaps(features, proj_t, coord, self.volume_aggregation_method, vol_conf)
        volumes = self.volume_net(volumes, v2v_conv, norm)
        kp, volumes = ops.integrate_tensor_3d_with_coordinates(volumes * self.volume_multiplier, coord, self.volume_softmax)
        return kp, features, volumes, vol_conf, coord


class AlgebraicTriangulationNet(_EngineOwner):
    """Drop-in for reference mvn/models/triangulation.py:131-200 (BASELINE config #5): backbone heatmaps -> 2-D
    soft-argmax -> confidence-weighted DLT.  Same ctor keys (`config.model.use_confidences`, `heatmap_softmax`,
    `heatmap_multiplier`, `backbone.*`), same config side effects, same 4-tuple.  backend="native": eval / no-grad on the
    kernels (engine.algebraic_forward); "torch": autograd torch ops; "hybrid": torch backbone, native 2-D soft-argmax and DLT
    with their backward kernels (trains, any mode)."""

    def __init__(self, config, device="cuda:0", backend=None, conv_mode=None, backbone_backend="torch", norm_backend="torch",
                 train_graph=False, head_backend="torch", eval_backend=None):
        super().__init__()
        self.use_confidences = config.model.use_confidences
        config.model.backbone.alg_confidences = False
        config.model.backbone.vol_confidences = False
        if self.use_confidences:
            config.model.backbone.alg_confidences = True
        self.backbone = pose_resnet.get_pose_net(config.model.backbone, device=device)
        self.heatmap_softmax = config.model.heatmap_softmax
        self.heatmap_multiplier = config.model.heatmap_multiplier
        self.backend = backend or os.environ.get("LT_B200_BACKEND", "native")
        self.conv_mode = conv_mode or os.environ.get("LT_B200_CONV", "tc")
        _check_backends(self.backend, self.conv_mode, backbone_backend, norm_backend, head_backend=head_backend, eval_backend=eval_backend)
        _check_train_graph(train_graph, self.backend)
        self.head_backend = head_backend
        self.eval_backend = eval_backend
        self.backbone_backend = backbone_backend
        self.norm_backend = norm_backend
        self.clone_outputs = True
        self._engine = None
        self._train_graphs = TrainGraphs() if train_graph else None

    def engine(self):
        if self._engine is None:
            from .engine import NativeEngine
            self._engine = NativeEngine(self, mode=self.conv_mode, use_graph=False)
        return self._engine

    def forward(self, images, proj_matricies, batch):
        if self.backend in ("torch", "hybrid") and not self._native_eval():
            # "hybrid": torch/cuDNN backbone with the native 2-D soft-argmax and DLT (forward + backward kernels) in the autograd graph
            if self.backend == "hybrid" and not images.is_cuda:
                raise RuntimeError("lt_b200 hybrid backend needs CUDA tensors (native custom ops); use backend='torch' on CPU")
            return self._run_device(self._forward_torch, (images, proj_matricies))
        return self._forward_native(images, proj_matricies)

    def _forward_native(self, images, proj_matricies):
        """The native engine's forward: backend="native" eagerly; the eval forwards of eval_backend="native" from one CUDA graph per
        input shape, with the volumetric model's clone_outputs semantics."""
        if not images.is_cuda:
            raise RuntimeError("lt_b200 native backend needs CUDA tensors; construct the model with backend='torch' for CPU/autograd")
        if self.training or torch.is_grad_enabled():
            raise RuntimeError("lt_b200 native backend is inference-only: use model.eval() under torch.no_grad(), or backend='torch'")
        H, W = images.shape[3:]
        if self.conv_mode != "simt" and (H % 2 or W % 2):      # the exact-fp32 mode's stem is an ordinary conv and takes odd sides
            raise ValueError("lt_b200 native backend needs even image sides (space-to-depth stem), got %dx%d" % (H, W))
        args = (images.float().contiguous(), proj_matricies.float().contiguous(), self.heatmap_multiplier, self.use_confidences,
                self.heatmap_softmax)
        with torch.cuda.device(images.device):
            if self.backend == "native":
                return self.engine().algebraic_forward(*args)
            outs = self.engine().algebraic_forward_graphed(*args)
        return tuple(o.clone() for o in outs) if self.clone_outputs else outs

    def _forward_torch(self, images, proj_matricies):
        """The reference forward on torch autograd, (images, proj_matricies) -> (kp3d, kp2d, heatmaps, alg_conf): everything runs on
        the device.  backend="hybrid" runs its 2-D soft-argmax and DLT on the native kernels."""
        ops_backend = "hybrid" if self.backend == "hybrid" else "torch"
        B, V = images.shape[:2]
        conv, _, norm = _hooks(self.backbone_backend, self.norm_backend)
        heatmaps, _, alg_conf, _ = self.backbone(images.reshape(-1, *images.shape[2:]), conv, norm, _head_tail(self.head_backend))
        if not self.use_confidences:
            alg_conf = torch.ones(B * V, heatmaps.shape[1], dtype=torch.float, device=images.device)
        kp2d, heatmaps = op.integrate_tensor_2d(heatmaps * self.heatmap_multiplier, self.heatmap_softmax, backend=ops_backend)
        heatmaps = heatmaps.view(B, V, *heatmaps.shape[1:])
        kp2d = kp2d.view(B, V, *kp2d.shape[1:])
        alg_conf = alg_conf.view(B, V, -1)
        if self.use_confidences and self.head_backend == "native":
            alg_conf = autograd_ops.view_normalize(alg_conf, 1e-5)
        else:
            alg_conf = alg_conf / alg_conf.sum(dim=1, keepdim=True) + 1e-5
        h, w = heatmaps.shape[3:]
        H, W = images.shape[3:]
        # the (W / w, H / h) scale is filled on the device: a host-to-device copy would synchronise and cannot be captured
        scale = torch.full((2,), W / w, device=images.device, dtype=kp2d.dtype)
        scale[1].fill_(H / h)
        kp2d = kp2d * scale
        kp3d = multiview.triangulate_batch_of_points(proj_matricies, kp2d, confidences_batch=alg_conf, backend=ops_backend)
        return kp3d, kp2d, heatmaps, alg_conf


def draw_view_pairs(batch_size, n_joints, n_views, n_iters):
    """(B, J, n_iters, 2) int32 view pairs, drawn with Python's global `random` in the reference's order (sample outer, joint
    inner, then the draws; triangulation.py:60-64, :84-85), each `sorted(random.sample(range(V), 2))`.  Python <= 3.10 sampled the
    reference's set of small ints as this range (later versions refuse a set), so after `random.seed(s)` the pairs, and
    `random.getstate()` afterwards, are the reference's."""
    views = range(n_views)
    pairs = np.empty((batch_size, n_joints, n_iters, 2), dtype=np.int32)
    for b in range(batch_size):
        for j in range(n_joints):
            for i in range(n_iters):
                pairs[b, j, i] = sorted(random.sample(views, 2))
    return pairs


def _dlt64(rows, mask):
    """rows (N, V, 2, 4) float64 DLT rows, mask (N, V) bool -> (N, 3): the smallest eigenvector of A^T A over the masked views."""
    A = (rows * mask[:, :, None, None]).reshape(rows.shape[0], -1, 4)
    u = torch.linalg.eigh(A.transpose(1, 2) @ A)[1][..., 0]
    return u[:, :3] / u[:, 3:]


def _project64(P, X):
    """pi(X) (N, V, 2) and the depth w (N, V, 1) of points X (N, 3) through P (N, V, 3, 4), float64 (multiview.py:89-110)."""
    uvw = torch.einsum("nvij,nj->nvi", P, torch.cat([X, torch.ones_like(X[:, :1])], 1))
    return uvw[..., :2] / uvw[..., 2:], uvw[..., 2:]


def _error2(P, pts, X):
    """(0.5 |p - pi(X)|)^2 per view, (N, V): the square of multiview.py:186-193's reprojection error."""
    return 0.25 * ((pts - _project64(P, X)[0]) ** 2).sum(-1)


def triangulate_ransac_batch(proj, keypoints_2d, pairs, reprojection_error_epsilon=15, direct_optimization=True, max_iters=1000):
    """Batched float64 torch formulation of triangulate_ransac (triangulation.py:72-128) over every (sample, joint) at once, on any
    device: proj (B, V, 3, 4), keypoints_2d (B, V, J, 2) int64, pairs (B, J, n_iters, 2) -> (keypoints_3d (B, J, 3) float64, inlier
    mask (B, J, V) bool).  The same steps as the native kernel (csrc/ransac.cu): pair DLTs, strict inlier test, first largest set,
    inlier DLT, and the Huber refinement by iteratively reweighted Levenberg-Marquardt."""
    B, V, J = keypoints_2d.shape[:3]
    N, n_iters = B * J, pairs.shape[2]
    dev = keypoints_2d.device
    P = proj.to(dev, torch.float64)[:, None].expand(B, J, V, 3, 4).reshape(N, V, 3, 4)
    pts = keypoints_2d.to(torch.float64).permute(0, 2, 1, 3).reshape(N, V, 2)
    rows = torch.stack([pts[..., 0:1] * P[:, :, 2] - P[:, :, 0], pts[..., 1:2] * P[:, :, 2] - P[:, :, 1]], dim=2)   # (N, V, 2, 4)
    ar = torch.arange(N, device=dev)
    pr = pairs.to(dev).reshape(N, n_iters, 2).long()
    best = torch.zeros((N, V), dtype=torch.bool, device=dev)
    best_n = torch.zeros(N, dtype=torch.long, device=dev)
    for i in range(n_iters):
        mask = torch.zeros((N, V), dtype=torch.bool, device=dev)
        mask[ar, pr[:, i, 0]] = True
        mask[ar, pr[:, i, 1]] = True
        mask = mask | (_error2(P, pts, _dlt64(rows, mask)).sqrt() < reprojection_error_epsilon)
        n = mask.sum(1)
        better = n > best_n
        best = torch.where(better[:, None], mask, best)
        best_n = torch.where(better, n, best_n)
    best = best | (best_n == 0)[:, None]               # the reference's "no inliers -> all views" (:100-101)
    X = _dlt64(rows, best)
    if direct_optimization:
        X = _refine_huber(P, pts, best, X, max_iters)
    return X.reshape(B, J, 3), best.reshape(B, J, V)


def _refine_huber(P, pts, mask, X, max_iters):
    """1/2 sum over the inliers of rho(f^2) (Huber, f_scale 1) minimised per item from X as ransac_refine (csrc/ransac.cu) does:
    weights 1 / max(f, 1) on the residual components, the Gauss-Newton curvature of f above f = 1, Marquardt damping, steps kept
    only where they lower the cost."""
    w_in = mask.to(X.dtype)

    def cost(X):
        z = _error2(P, pts, X)
        return 0.5 * (torch.where(z <= 1, z, 2 * z.sqrt() - 1) * w_in).sum(1)

    c = cost(X)
    active = torch.isfinite(c)
    lam = torch.full_like(c, 1e-3)
    for _ in range(max_iters):
        if not bool(active.any()):
            break
        puv, w = _project64(P, X)
        r = 0.5 * (puv - pts)                                                            # (N, V, 2)
        f = r.norm(dim=-1)
        outer = f > 1
        wt = torch.where(outer, 1 / f, torch.ones_like(f)) * w_in
        Jac = 0.5 * (P[:, :, :2, :3] - puv[..., None] * P[:, :, 2:3, :3]) / w[..., None]  # (N, V, 2, 3)
        jtr = torch.einsum("nvai,nva->nvi", Jac, r)
        jr = torch.where(outer[..., None], jtr / f[..., None], torch.zeros_like(jtr))      # radial direction of the Huber branch
        H = torch.einsum("nv,nvai,nvaj->nij", wt, Jac, Jac) - torch.einsum("nv,nvi,nvj->nij", wt, jr, jr)
        g = torch.einsum("nv,nvi->ni", wt, jtr)
        A = H + torch.diag_embed(lam[:, None] * torch.diagonal(H, dim1=1, dim2=2))
        d = -torch.linalg.solve_ex(A, g[..., None])[0][..., 0]
        Xn = X + d
        cn = cost(Xn)
        acc = active & (cn < c)
        X = torch.where(acc[:, None], Xn, X)
        c = torch.where(acc, cn, c)
        lam = torch.where(acc, (lam * 0.1).clamp(min=1e-12), lam * 10)
        done = acc & (d.norm(dim=1) <= 1e-12 * X.norm(dim=1))
        active = active & ~done & ~(~acc & (lam > 1e16))
    return X


class RANSACTriangulationNet(_EngineOwner):
    """Drop-in for reference mvn/models/triangulation.py:17-128 (the "ransac" model of train.py): raw backbone heat maps -> arg-max
    key points -> per-(sample, joint) RANSAC over view pairs, the inlier DLT and, with `config.model.direct_optimization`, the Huber
    refinement of the reprojection error.  Same ctor keys, config side effects, `backbone` attribute, state_dict keys and 4-tuple.
    The view pairs are drawn on the host with Python's `random` in the reference's order (draw_view_pairs).
    backend="native": eval / no-grad on the kernels (engine.ransac_forward); "torch": the torch backbone and the batched float64
    formulation triangulate_ransac_batch (CPU or GPU).  Neither trains through the RANSAC, as the reference does not."""

    n_iters = 10                        # triangulate_ransac's defaults (:72)
    reprojection_error_epsilon = 15

    def __init__(self, config, device="cuda:0", backend=None, conv_mode=None):
        super().__init__()
        config.model.backbone.alg_confidences = False      # the reference mutates the caller's config here (:21-23); so do we
        config.model.backbone.vol_confidences = False
        self.backbone = pose_resnet.get_pose_net(config.model.backbone, device=device)
        self.direct_optimization = config.model.direct_optimization
        self.backend = backend or os.environ.get("LT_B200_BACKEND", "native")
        if self.backend not in ("native", "torch"):
            raise ValueError("unknown backend {!r} (RANSACTriangulationNet has 'native' and 'torch')".format(self.backend))
        self.conv_mode = conv_mode or os.environ.get("LT_B200_CONV", "tc")
        self._engine = None
        self._train_graphs = None

    def engine(self):
        if self._engine is None:
            from .engine import NativeEngine
            self._engine = NativeEngine(self, mode=self.conv_mode, use_graph=False)
        return self._engine

    def forward(self, images, proj_matricies, batch):
        B, V = images.shape[:2]
        assert V >= 2                                       # triangulate_ransac (:74), before anything is drawn
        if self.backend == "torch":
            return self._forward_torch(images, proj_matricies)
        if not images.is_cuda:
            raise RuntimeError("lt_b200 native backend needs CUDA tensors; construct the model with backend='torch' for CPU/autograd")
        if self.training or torch.is_grad_enabled():
            raise RuntimeError("lt_b200 native backend is inference-only: use model.eval() under torch.no_grad(), or backend='torch'")
        H, W = images.shape[3:]
        if H % 2 or W % 2:
            raise ValueError("lt_b200 native backend needs even image sides (space-to-depth stem), got %dx%d" % (H, W))
        dev = images.device
        pairs = draw_view_pairs(B, self.backbone.num_joints, V, self.n_iters)
        with torch.cuda.device(dev):
            pairs_t, = _upload(dev, pairs, dtype=torch.int32)
            return self.engine().ransac_forward(images.float().contiguous(), proj_matricies.to(dev, torch.float32).contiguous(), pairs_t,
                                                self.n_iters, self.reprojection_error_epsilon, self.direct_optimization)

    def _forward_torch(self, images, proj_matricies):
        """The reference forward with the batched torch RANSAC: -> (keypoints_3d, keypoints_2d int64, heatmaps, confidences)."""
        B, V = images.shape[:2]
        H, W = images.shape[3:]
        dev = images.device
        heatmaps, _, _, _ = self.backbone(images.reshape(-1, *images.shape[2:]), layers.torch_conv, layers.torch_norm)
        J, h, w = heatmaps.shape[1:]
        heatmaps = heatmaps.view(B, V, J, h, w)
        _, idx = torch.max(heatmaps.view(B, V, J, -1), dim=-1)                  # :45-52
        kp = torch.stack([idx % w, idx // w], dim=-1)
        keypoints_2d = torch.zeros_like(kp)
        keypoints_2d[..., 0] = kp[..., 0] * (W / w)
        keypoints_2d[..., 1] = kp[..., 1] * (H / h)
        pairs = torch.from_numpy(draw_view_pairs(B, J, V, self.n_iters))
        kp3d, _ = triangulate_ransac_batch(proj_matricies, keypoints_2d.detach(), pairs, self.reprojection_error_epsilon,
                                           self.direct_optimization)
        confidences = torch.zeros((B, V, J), dtype=torch.float32, device=dev)   # :59, the "plug"
        return kp3d.float(), keypoints_2d, heatmaps, confidences


class LazyCuboids(collections.abc.Sequence):
    """The per-sample volumetric.Cuboid3D of a TwoStageTriangulationNet forward, built on first access.  That access copies the
    device base points to the host, the forward's only synchronisation, paid only by a caller that reads the cuboids (e.g. for
    visualisation).  The positions are base - side / 2 in float64 from those float32 base points, as _host_geometry forms them from
    the same key points, so each Cuboid3D equals the two-pass protocol's."""

    def __init__(self, base_points, cuboid_side):
        self._base = base_points
        self._side = cuboid_side
        self._items = None

    def _built(self):
        if self._items is None:
            base = self._base.cpu().numpy().astype(np.float64)
            self._items = _place_cuboids(base, np.array([self._side] * 3, dtype=np.float64))[1]
            self._base = None
        return self._items

    def __len__(self):
        return self._base.shape[0] if self._items is None else len(self._items)

    def __getitem__(self, i):
        return self._built()[i]


class TwoStageTriangulationNet(_EngineOwner):
    """The volumetric model without ground truth: each sample's cuboid is placed at the pelvis of an algebraic model's key points,
    on the device.  This is the reference's two-stage protocol (evaluate AlgebraicTriangulationNet, reload its results file as
    batch['pred_keypoints_3d'] for a volumetric config with use_gt_pelvis: false) without the host round trip between the stages.

    forward(images, proj_matricies, batch) returns the volumetric model's 7-tuple.  proj_matricies are the image-space matrices the
    algebraic model takes; None derives them from batch['cameras'] as prepare_batch does.  The volumetric stage keeps its host geometry
    from batch['cameras'].  The algebraic forward, the hand-off (lt_cuboid_from_keypoints_fwd) and the volumetric device forward replay
    from one CUDA graph per input shape, re-captured when either model's packed weights go stale.  `base_points` is the device pelvis;
    `cuboids` is a LazyCuboids.  Native backend, inference only."""

    def __init__(self, algebraic, volumetric):
        super().__init__()
        if not isinstance(algebraic, AlgebraicTriangulationNet) or not isinstance(volumetric, VolumetricTriangulationNet):
            raise ValueError("TwoStageTriangulationNet takes an AlgebraicTriangulationNet and a VolumetricTriangulationNet (got %s, %s)"
                             % (type(algebraic).__name__, type(volumetric).__name__))
        for name, m in (("algebraic", algebraic), ("volumetric", volumetric)):
            if m.backend != "native":
                raise ValueError("TwoStageTriangulationNet runs the native backend only; the %s model has backend=%r" % (name, m.backend))
        devices = {str(t.device) for m in (algebraic, volumetric) for t in m.parameters()}
        if len(devices) != 1:
            raise ValueError("both models must live on one device (got %s)" % ", ".join(sorted(devices)))
        if algebraic.backbone.num_joints != volumetric.num_joints:
            raise ValueError("the models predict different joint counts (algebraic %d, volumetric %d)"
                             % (algebraic.backbone.num_joints, volumetric.num_joints))
        if volumetric.use_gt_pelvis:
            raise ValueError("the volumetric model has use_gt_pelvis=True; the two-stage model places its cuboids at the algebraic "
                             "model's pelvis, so it needs a model configured with use_gt_pelvis=False")
        if volumetric.kind not in capi.KIND:
            raise ValueError("unknown skeleton kind {!r} (mpii or coco)".format(volumetric.kind))
        pelvis_joint = 12 if volumetric.kind == "coco" else 6
        if volumetric.num_joints <= pelvis_joint:
            raise ValueError("skeleton kind %r reads joint %d, but the models predict %d joints"
                             % (volumetric.kind, pelvis_joint, volumetric.num_joints))
        self.algebraic = algebraic
        self.volumetric = volumetric
        self.training = algebraic.training or volumetric.training      # the mode of the models it was given; .eval() sets all three
        self.clone_outputs = True
        self._graphs = {}

    def _invalidate_engine(self):
        self._graphs = {}
        self.algebraic._invalidate_engine()
        self.volumetric._invalidate_engine()

    def forward(self, images, proj_matricies, batch):
        if self.algebraic.training or self.volumetric.training or torch.is_grad_enabled():
            raise RuntimeError("TwoStageTriangulationNet is inference-only: call model.eval() under torch.no_grad()")
        if not images.is_cuda:
            raise RuntimeError("TwoStageTriangulationNet runs the native backend: it needs CUDA tensors (got %s)" % images.device)
        dev = images.device
        if next(self.parameters()).device != dev:
            raise RuntimeError("the images are on %s, the models on %s" % (dev, next(self.parameters()).device))
        B = images.shape[0]
        H, W = images.shape[3:]
        if H % 2 or W % 2:
            raise ValueError("lt_b200 native backend needs even image sides (space-to-depth stem), got %dx%d" % (H, W))
        hm_shape = (backbone_map_size(H), backbone_map_size(W))
        proj_hm, _, step, rots = self.volumetric._pelvis_free_geometry(batch, B, (H, W), hm_shape)
        host = (proj_hm, step, rots.reshape(B, 9))
        if proj_matricies is None:
            host += (multiview.stack_projections(batch["cameras"]),)                # datasets/utils.py:61-63
        with torch.cuda.device(dev):
            up = _upload(dev, *host)
            proj_img = up[3] if proj_matricies is None else proj_matricies.to(dev, torch.float32).contiguous()
            outs = self._replay(images.float().contiguous(), proj_img, *up[:3])
        if self.clone_outputs:
            outs = tuple(o.clone() for o in outs)
        center, kp, features, volumes, coord = outs[:5]
        if tuple(features.shape[3:]) != hm_shape:
            raise RuntimeError("feature map %s differs from the heat-map size %s used for the projection matrices"
                               % (tuple(features.shape[3:]), hm_shape))
        vol_conf = outs[5] if len(outs) > 5 else None
        cuboids = LazyCuboids(center if self.clone_outputs else center.clone(), self.volumetric.cuboid_side)
        return kp, features, volumes, vol_conf, cuboids, coord, center

    def _replay(self, *inputs):
        """_device_forward(*inputs) replayed from the graph of this input shape; captured on a miss or when either engine's packed
        weights are stale.  -> the graph's static outputs."""
        version = (self.algebraic.engine()._param_version(), self.volumetric.engine()._param_version())
        key = (tuple(inputs[0].shape), inputs[0].device)
        entry = self._graphs.get(key)
        if entry is None or entry[0] != version:
            self._graphs.pop(key, None)                  # free the stale graph's memory before capturing its successor
            entry = self._graphs[key] = (version,) + self._capture(inputs)
        _, graph, static_in, static_out = entry
        for dst, src in zip(static_in, inputs):
            dst.copy_(src, non_blocking=True)
        graph.replay()
        return static_out

    def _capture(self, inputs):
        self.algebraic.engine().prepare()
        self.volumetric.engine().prepare()
        static_in = [t.clone() for t in inputs]
        side = torch.cuda.Stream(device=inputs[0].device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._device_forward(*static_in)     # warm-up: module loads, function attributes, the soft-argmax grid
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_out = self._device_forward(*static_in)
        return graph, static_in, static_out

    def _device_forward(self, images, proj_img, proj_hm, step, rot):
        """Both stages and the hand-off on the device: (images, image-space and heat-map-space projections, voxel step, rotations
        (B, 9)) -> (base points, kp, features, volumes, coord[, vol_conf])."""
        a, v = self.algebraic, self.volumetric
        kp_alg = a.engine().algebraic_forward(images, proj_img, a.heatmap_multiplier, a.use_confidences, a.heatmap_softmax)[0]
        center = torch.empty((images.shape[0], 3), dtype=torch.float32, device=images.device)
        position = torch.empty_like(center)
        capi.cuboid_from_keypoints(kp_alg, v.kind, v.cuboid_side, center, position)
        return (center,) + tuple(v.engine()._device_forward(images, proj_hm, position, center, step, rot))
