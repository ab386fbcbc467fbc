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
import os

import numpy as np
import torch
from torch import nn

from . import autograd_ops, layers, multiview, op, pose_resnet, torch_ops, volumetric
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


_NO_V2V = object()      # the v2v_backend of a model without a V2V net (None stays an unknown v2v_backend)


def _check_backends(backend, conv_mode, backbone_backend, norm_backend, v2v_backend=_NO_V2V):
    """ValueError unless the training switches are known values in a supported combination.

    v2v_backend="native" / backbone_backend="native": every Conv3d / ConvTranspose3d of volume_net / every Conv2d / ConvTranspose2d
    of the backbone, its confidence heads and `process_features` runs forward, data gradient and weight gradient on the native
    tensor-core kernels.  Both need backend="hybrid" and conv_mode="tc".
    norm_backend="native": every BatchNorm2d / BatchNorm3d of the backbone, its confidence heads and the V2V net, fused with the ReLU
    after it and the residual add of a residual unit, trains on the native kernels.  The kernels read the channels-last maps the
    native convolutions produce, so it needs backend="hybrid" and every conv switch of the model "native"."""
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


def _hooks(backbone_backend, norm_backend, v2v_backend="torch"):
    """(backbone conv, V2V conv, norm) hooks of checked switches: the torch formulas in layers.py for "torch", autograd_ops'
    native training functions for "native"."""
    return (autograd_ops.backbone_conv if backbone_backend == "native" else layers.torch_conv,
            autograd_ops.v2v_conv if v2v_backend == "native" else layers.torch_conv,
            autograd_ops.batch_norm if norm_backend == "native" else layers.torch_norm)


def _upload(device, *arrays):
    """float32 tensors on `device` of host arrays (float64 cast last): on CUDA through one page-locked buffer and one asynchronous
    copy, so the host part of a forward does not wait for the device."""
    flat = [torch.from_numpy(np.ascontiguousarray(a)).float().reshape(-1) for a in arrays]
    host = torch.cat(flat)
    if device.type == "cuda":
        host = host.pin_memory().to(device, non_blocking=True)
    return tuple(t.view(a.shape) for t, a in zip(host.split([f.numel() for f in flat]), arrays))


def _check_train_graph(train_graph, backend):
    if train_graph and backend != "hybrid":
        raise ValueError("train_graph=True needs backend='hybrid' (got %r)" % (backend,))


class _EngineOwner(nn.Module):
    """Keeps the native engine's packed filters / CUDA graphs and the training graphs (train_graph.TrainGraphs) in step with the
    module's tensors: `.to()/.cuda()/.float()` (`_apply`) and `load_state_dict` invalidate them explicitly (tensor versions alone
    miss `p.data` updates)."""

    def _invalidate_engine(self):
        eng = self.__dict__.get("_engine")
        if eng is not None:
            eng.invalidate()
        graphs = self.__dict__.get("_train_graphs")
        if graphs is not None:
            graphs.invalidate()

    def _run_device(self, fn, inputs):
        """fn(*inputs): the device part of the forward, replayed from CUDA graphs with train_graph=True in a training forward."""
        if self._train_graphs is not None and self.training and torch.is_grad_enabled():
            return self._train_graphs.run(self, fn, inputs, self.clone_outputs)
        return fn(*inputs)

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
                 backbone_backend="torch", norm_backend="torch", train_graph=False):
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
        _check_backends(self.backend, self.conv_mode, backbone_backend, norm_backend, v2v_backend)
        _check_train_graph(train_graph, self.backend)
        self.v2v_backend = v2v_backend
        self.backbone_backend = backbone_backend
        self.norm_backend = norm_backend
        self.use_cuda_graph = use_cuda_graph
        self.clone_outputs = True
        self._engine = None
        self._train_graphs = TrainGraphs() if train_graph else None

    # ---------------------------------------------------------------- host-side geometry
    def _host_geometry(self, batch, batch_size, image_shape, heatmap_shape):
        proj = multiview.stack_projections(batch["cameras"], image_shape, heatmap_shape)      # (B, V, 3, 4) f32
        base = _base_points(batch, batch_size, self.kind, self.use_gt_pelvis)                 # (B, 3) f64
        sides = np.array([self.cuboid_side] * 3, dtype=np.float64)
        position = base - sides / 2
        cuboids = [volumetric.Cuboid3D(position[b], sides) for b in range(batch_size)]
        axis = [0, 1, 0] if self.kind == "coco" else [0, 0, 1]
        rots = np.empty((batch_size, 3, 3), dtype=np.float64)
        for b in range(batch_size):
            theta = np.random.uniform(0.0, 2 * np.pi) if self.training else 0.0   # triangulation.py:318-321
            rots[b] = volumetric.get_rotation_matrix(axis, theta)
        step = sides / (self.volume_size - 1)
        return proj, base, position, step, rots, cuboids

    def engine(self):
        if self._engine is None:
            from .engine import NativeEngine
            self._engine = NativeEngine(self, mode=self.conv_mode, use_graph=self.use_cuda_graph)
        return self._engine

    # ---------------------------------------------------------------- forward
    def forward(self, images, proj_matricies, batch):
        if self.backend in ("torch", "hybrid"):
            # "hybrid": torch/cuDNN convolutions with the native custom ops (forward + backward kernels) in the autograd graph
            return self._forward_torch(images, batch)
        if self.backend != "native":
            raise ValueError("unknown backend {!r}".format(self.backend))
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

        def up(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev, non_blocking=True)

        with torch.cuda.device(dev):      # launches go to the model's device, whatever the caller's current device is
            outs = self.engine().forward(
                images.float().contiguous(), up(proj), up(position), up(base), up(step), up(rots.reshape(B, 9)))
            base_points = up(base)
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
        heatmaps, features, _, vol_conf = self.backbone(flat, conv, norm)
        hm_shape = (backbone_map_size(images.shape[3]), backbone_map_size(images.shape[4]))
        if tuple(heatmaps.shape[2:]) != hm_shape:
            raise RuntimeError("heat-map size %s differs from the size %s used for the projection matrices"
                               % (tuple(heatmaps.shape[2:]), hm_shape))
        if vol_conf is not None:
            vol_conf = vol_conf.view(B, V, *vol_conf.shape[1:])
            if self.volume_aggregation_method == "conf_norm":
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
                 train_graph=False):
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
        _check_backends(self.backend, self.conv_mode, backbone_backend, norm_backend)
        _check_train_graph(train_graph, self.backend)
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
        if self.backend == "torch":
            return self._forward_torch(images, proj_matricies)
        if self.backend == "hybrid":
            # torch/cuDNN backbone with the native 2-D soft-argmax and DLT (forward + backward kernels) in the autograd graph
            if not images.is_cuda:
                raise RuntimeError("lt_b200 hybrid backend needs CUDA tensors (native custom ops); use backend='torch' on CPU")
            return self._run_device(self._forward_torch, (images, proj_matricies))
        if not images.is_cuda:
            raise RuntimeError("lt_b200 native backend needs CUDA tensors; construct the model with backend='torch' for CPU/autograd")
        if self.training or torch.is_grad_enabled():
            raise RuntimeError("lt_b200 native backend is inference-only: use model.eval() under torch.no_grad(), or backend='torch'")
        with torch.cuda.device(images.device):
            return self.engine().algebraic_forward(images.float().contiguous(), proj_matricies.float().contiguous(),
                                                   self.heatmap_multiplier, self.use_confidences, self.heatmap_softmax)

    def _forward_torch(self, images, proj_matricies):
        """The reference forward on torch autograd, (images, proj_matricies) -> (kp3d, kp2d, heatmaps, alg_conf): everything runs on
        the device.  backend="hybrid" runs its 2-D soft-argmax and DLT on the native kernels."""
        ops_backend = "hybrid" if self.backend == "hybrid" else "torch"
        B, V = images.shape[:2]
        conv, _, norm = _hooks(self.backbone_backend, self.norm_backend)
        heatmaps, _, alg_conf, _ = self.backbone(images.reshape(-1, *images.shape[2:]), conv, norm)
        if not self.use_confidences:
            alg_conf = torch.ones(B * V, heatmaps.shape[1], dtype=torch.float, device=images.device)
        kp2d, heatmaps = op.integrate_tensor_2d(heatmaps * self.heatmap_multiplier, self.heatmap_softmax, backend=ops_backend)
        heatmaps = heatmaps.view(B, V, *heatmaps.shape[1:])
        kp2d = kp2d.view(B, V, *kp2d.shape[1:])
        alg_conf = alg_conf.view(B, V, -1)
        alg_conf = alg_conf / alg_conf.sum(dim=1, keepdim=True) + 1e-5
        h, w = heatmaps.shape[3:]
        H, W = images.shape[3:]
        # the (W / w, H / h) scale is filled on the device: a host-to-device copy would synchronise and cannot be captured
        scale = torch.full((2,), W / w, device=images.device, dtype=kp2d.dtype)
        scale[1].fill_(H / h)
        kp2d = kp2d * scale
        kp3d = multiview.triangulate_batch_of_points(proj_matricies, kp2d, confidences_batch=alg_conf, backend=ops_backend)
        return kp3d, kp2d, heatmaps, alg_conf
