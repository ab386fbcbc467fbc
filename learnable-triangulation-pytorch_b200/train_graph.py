"""CUDA-graph capture of hybrid training forwards (`train_graph=True`): one captured forward and one captured backward per step.

A model's forward splits into a host part (camera geometry, the random rotation draw, their upload) and a device function of tensors.
`TrainGraphs.run` replays the device function and its backward from two CUDA graphs, so a step costs a handful of host calls instead
of one Python hook, autograd node and ctypes call per layer.  The kernels are the ones the eager step runs; nothing is recomputed or
re-ordered, so results match the eager step within its own run-to-run spread.

Capture rules:
- One cache entry per input shapes / dtypes / device, parameter `requires_grad` mask, module training flags and the data_ptr of
  every parameter and buffer (the graphs read them at fixed addresses; `p.data = ...` moves one without a version bump).
- A miss runs the device function and its backward eagerly on a side stream (torch.autograd.grad, so `.grad` is untouched): module
  loads, kernel attributes, per-stream library workspaces and the native scratch buffers (autograd_ops._WORKSPACE,
  engine.splitk_workspace) are settled before capture.  Every BatchNorm's running buffers and num_batches_tracked are restored after
  capture, so the first replay is the step's one update.
- Both graphs go into one private memory pool per model, shared by all its captures: activations stay resident between steps.
  thread_local capture mode (a DataLoader's pin-memory thread makes CUDA calls meanwhile); anomaly mode off (its NaN checks read
  the device).  A failed capture raises RuntimeError; there is no eager fallback.
- Replay copies the inputs into the entry's static buffers, replays the forward and hands the outputs to autograd through one node.
  Its backward copies the output gradients into static buffers (zeros for outputs without one), replays the backward and returns
  the parameter gradients from one fresh buffer, which AccumulateGrad (and DDP's hooks) then take as usual.
"""
import warnings
import weakref

import torch
from torch import nn

from . import autograd_ops, engine


class _Entry:
    __slots__ = ("fwd", "bwd", "static_in", "outs", "layout", "diff", "gouts", "gout_zero", "params", "grad_shapes", "flat", "keep")


class _Replay(torch.autograd.Function):
    """Forward: replay the captured forward; backward: replay the captured backward.  The differentiable inputs are the parameters."""

    @staticmethod
    def forward(ctx, graphs, entry, clone, *params):
        entry.fwd.replay()
        graphs.replays += 1
        ctx.graphs, ctx.entry, ctx.replay = graphs, entry, graphs.replays
        ctx.set_materialize_grads(False)
        outs = tuple(o.clone() if clone else o.detach() for o in entry.outs)
        ctx.mark_non_differentiable(*[o for o, d in zip(outs, entry.diff) if not d])
        return outs

    @staticmethod
    def backward(ctx, *grads):
        e = ctx.entry
        if ctx.replay != ctx.graphs.replays:
            raise RuntimeError("train_graph: another training forward of this model ran before this backward and overwrote the "
                               "activations it needs; run backward before the next training forward")
        i = 0
        for g, d in zip(grads, e.diff):
            if not d:
                continue
            if g is not None:
                e.gouts[i].copy_(g)
                e.gout_zero[i] = False
            elif not e.gout_zero[i]:
                e.gouts[i].zero_()
                e.gout_zero[i] = True
            i += 1
        e.bwd.replay()
        out = [None] * len(e.params)
        if e.flat is not None:
            flat = e.flat.clone()
            off = 0
            for j, shape in enumerate(e.grad_shapes):
                if shape is not None:
                    n = shape.numel()
                    out[j] = flat[off:off + n].view(shape)
                    off += n
        return (None, None, None) + tuple(out)


def _norm_state(model):
    """Every BatchNorm running buffer and num_batches_tracked of the model (what a train-mode forward writes)."""
    return [b for m in model.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)
            for b in (m.running_mean, m.running_var, m.num_batches_tracked) if b is not None]


class TrainGraphs:
    """The training graphs of one model.  `captures` counts the (forward, backward) pairs captured so far."""

    def __init__(self):
        self.captures = 0
        self.replays = 0           # forward replays: a backward refuses to run once a later forward has replaced its activations
        self._entries = {}
        self._pool = None

    def invalidate(self):
        self._entries.clear()
        self._pool = None

    def run(self, model, fn, inputs, clone_outputs):
        """fn(*inputs) -> tuple of tensors or None, replayed from CUDA graphs; the outputs carry gradients to model's parameters."""
        if any(t.requires_grad for t in inputs):
            raise ValueError("train_graph: the captured backward computes parameter gradients only; the inputs must not require grad")
        params = list(model.parameters())
        key = _model_key(model, inputs)
        entry = self._entries.get(key)
        if entry is None:
            entry = self._entries[key] = self._capture(model, fn, inputs, params)
            self.captures += 1
        for dst, src in zip(entry.static_in, inputs):
            dst.copy_(src)
        outs = iter(_Replay.apply(self, entry, clone_outputs, *entry.params))
        return tuple(next(outs) if present else None for present in entry.layout)

    def _capture(self, model, fn, inputs, params):
        e = _Entry()
        e.params = [p for p in params if p.requires_grad]
        e.static_in = [t.detach().clone() for t in inputs]

        def warm_up():
            outs = fn(*e.static_in)
            diff = [o for o in outs if o is not None and o.requires_grad]
            torch.autograd.grad(diff, e.params, [torch.zeros_like(o) for o in diff], allow_unused=True)

        def capture(graph):
            e.fwd, e.bwd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with graph(e.fwd):
                outs = fn(*e.static_in)
            present = [o for o in outs if o is not None]
            e.diff = [o.requires_grad for o in present]
            diff = [o for o in present if o.requires_grad]
            e.gouts = [torch.zeros_like(o) for o in diff]
            e.gout_zero = [True] * len(diff)
            with graph(e.bwd):
                grads = torch.autograd.grad(diff, e.params, e.gouts, allow_unused=True)
                used = [g.reshape(-1) for g in grads if g is not None]
                e.flat = torch.cat(used) if used else None
            e.grad_shapes = [None if g is None else g.shape for g in grads]
            e.outs = [o.detach() for o in present]
            e.layout = [o is not None for o in outs]

        _capture_on_side_stream(self, inputs[0].device, _norm_state(model), warm_up, capture, "train_graph")
        e.keep = _captured_scratch()
        return e


def _model_key(model, inputs):
    """What a graph of `model`'s step depends on besides the values it reads: input shapes / dtypes / devices, the parameters'
    requires_grad mask, the data_ptr of every parameter and buffer, the modules' training flags, and whether
    torch.use_deterministic_algorithms is on (it selects the fixed-order backward kernels)."""
    params = list(model.parameters())
    return (tuple((tuple(t.shape), t.dtype, t.device) for t in inputs), tuple(p.requires_grad for p in params),
            tuple(p.data_ptr() for p in params), tuple(b.data_ptr() for b in model.buffers()),
            tuple(m.training for m in model.modules()), torch.are_deterministic_algorithms_enabled())


def _capture_on_side_stream(cache, dev, state, warm_up, capture, what, reset=None):
    """warm_up() eagerly on a side stream, then capture(graph) there, where graph(g) is the capture context of CUDAGraph g in
    cache's private pool (created on first use), thread_local mode.  Anomaly mode is off throughout.  The tensors of `state` are
    copied back afterwards, on the caller's stream, to their values before the warm-up; reset(), if given, runs after them.  A
    failure raises RuntimeError naming `what`; nothing falls back to eager."""
    saved = [b.clone() for b in state]
    cur = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(cur)
    try:
        with torch.cuda.device(dev), torch.autograd.set_detect_anomaly(False), torch.cuda.stream(side):
            warm_up()
            if cache._pool is None:
                cache._pool = torch.cuda.graph_pool_handle()
            capture(lambda g: torch.cuda.graph(g, pool=cache._pool, stream=side, capture_error_mode="thread_local"))
    except Exception as exc:
        raise RuntimeError("%s: capturing the training step failed: %s: %s" % (what, type(exc).__name__, exc)) from exc
    finally:
        cur.wait_stream(side)
        with torch.cuda.stream(cur):
            for b, s in zip(state, saved):
                b.copy_(s)
            if reset is not None:
                reset()


def _captured_scratch():
    """The scratch buffers captured launches write at fixed addresses: an entry keeps them, so that an eager call that grows a
    workspace later does not free memory a graph still uses."""
    return list(autograd_ops._WORKSPACE.values()) + list(engine._SPLITK_WS.values())


_CRITERIA = {"MSE": "mse", "MSESmooth": "mse_smooth", "MAE": "mae"}       # train.py:416-425
_BASE_JOINT = {"human36m": 6, "coco": 11}                                 # the 1-view transform's base joint, train.py:200-205


class _StepEntry:
    __slots__ = ("graph", "static_in", "outs", "metrics", "grads", "keep")


def _hashable(v):
    return v.data_ptr() if torch.is_tensor(v) else tuple(v) if isinstance(v, list) else v


class TrainStep:
    """One training iteration of the reference's train.py (train.py:185-263) replayed from one CUDA graph.

        step = TrainStep(model, optimizer, config)
        outputs, metrics = step(*dataset_utils.prepare_batch(batch, device, config), batch)

    `model` is an AlgebraicTriangulationNet or VolumetricTriangulationNet with backend="hybrid" (any conv / norm switches; its own
    train_graph graphs are not used), `optimizer` a torch.optim.Adam with capturable=True in every param group, `config` the
    experiment config train.py loads.  `outputs` is the model's tuple; `metrics` maps the keys of train.py's metric_dict
    (config.opt.criterion, "volumetric_ce_loss" with use_volumetric_ce_loss, "total_loss", "grad_norm_times_lr", "l2" and, for the
    volumetric model, "base_point_l2") to 0-dim device tensors.  Nothing is read back to the host.

    What a call does, as train.py: validity binarised (> 0); on a 1-view batch the key points relative to the base joint (6 for
    config.kind "human36m", 11 for "coco"; another kind raises ValueError); the criterion (the native one of lt_b200.loss) on key
    points scaled by scale_keypoints_3d; the cross-entropy loss (loss.volumetric_ce_loss) on the unscaled ground truth, weighted;
    backward of the total; clip_grad_norm_(model.parameters(), grad_clip / lr) when config.opt has grad_clip; lr times the norm of
    the trainable parameters' gradients after clipping (float64 sum of the per-parameter norms); optimizer.step(); the L2 metric;
    base_point_l2 from config.model.kind (mpii: joint 6 of the ground truth; coco: the midpoint of joints 11 and 12, where the
    reference raises NameError, train.py:256).  The config is read once, here.

    The host part stays eager (the volumetric model's camera geometry, rotation draw and upload).  Everything else -- the model's
    device function, the transform and scaling, the losses and metrics, torch.autograd.backward, the clipping, the gradient norm and
    optimizer.step() -- is one graph, captured with PyTorch's whole-network pattern: the gradients live in the graph's pool, and
    after each call every trainable parameter's .grad is that step's (clipped) gradient (zero_grad() between steps is allowed and
    not needed).  A graph is captured per input shapes, requires_grad mask, training flags, parameter / buffer / optimizer-state
    data_ptrs and param-group hyperparameters (a capturable Adam bakes its float lr into the graph, so changing lr recaptures, as do
    opt.load_state_dict and model.to()); a capture replaces the graphs of the same input shapes.  A capture first runs the whole
    step eagerly on a side stream and then restores the parameters, the optimizer state (a state that was empty goes back to zeros
    and step 0) and every BatchNorm buffer, so the first replay is the first update.  `captures` counts captures.  clone_outputs
    False returns the graph's own output and metric buffers, valid until the next call.  Every call invalidates the model's native
    engine, so an eval_backend="native" forward after it re-packs the updated weights.

    DistributedDataParallel is not supported (the gradient all-reduce would have to run inside the graph)."""

    def __init__(self, model, optimizer, config, clone_outputs=True):
        from .triangulation import AlgebraicTriangulationNet, VolumetricTriangulationNet
        if isinstance(model, nn.parallel.DistributedDataParallel):
            raise ValueError("TrainStep does not take a DistributedDataParallel model: its gradient all-reduce cannot run inside "
                             "the step's graph; pass the module itself")
        if isinstance(model, VolumetricTriangulationNet):
            name = "vol"
        elif isinstance(model, AlgebraicTriangulationNet):
            name = "alg"
        else:
            raise ValueError("TrainStep takes an AlgebraicTriangulationNet or a VolumetricTriangulationNet (got %s)"
                             % type(model).__name__)
        if model.backend != "hybrid":
            raise ValueError("TrainStep needs a model with backend='hybrid' (got %r)" % (model.backend,))
        if config.model.name != name:
            raise ValueError("config.model.name is %r but the model is a %s (%r)" % (config.model.name, type(model).__name__, name))
        if not isinstance(optimizer, torch.optim.Adam) or not all(g.get("capturable", False) for g in optimizer.param_groups):
            raise ValueError("TrainStep needs torch.optim.Adam with capturable=True in every param group (its step runs inside the "
                             "graph), got %s" % type(optimizer).__name__)
        opt = config.opt
        if opt.criterion not in _CRITERIA:
            raise ValueError("unknown criterion %r (MSE, MSESmooth or MAE)" % (opt.criterion,))
        self.use_ce = opt.use_volumetric_ce_loss if hasattr(opt, "use_volumetric_ce_loss") else False
        if self.use_ce and name != "vol":
            raise ValueError("use_volumetric_ce_loss needs the volumetric model")
        if name == "vol" and config.model.kind not in ("mpii", "coco"):
            raise ValueError("base_point_l2 needs config.model.kind 'mpii' or 'coco' (got %r)" % (config.model.kind,))
        self.model, self.optimizer, self.clone_outputs = model, optimizer, clone_outputs
        self.volumetric = name == "vol"
        self.criterion = opt.criterion
        self.kind = _CRITERIA[opt.criterion]
        self.threshold = float(opt.mse_smooth_threshold) if opt.criterion == "MSESmooth" else 400.0
        self.scale = opt.scale_keypoints_3d if hasattr(opt, "scale_keypoints_3d") else 1.0
        self.ce_weight = opt.volumetric_ce_loss_weight if hasattr(opt, "volumetric_ce_loss_weight") else 1.0
        self.lr = opt.lr
        self.grad_clip = opt.grad_clip if hasattr(opt, "grad_clip") else None
        self.base_joint = _BASE_JOINT.get(config.kind) if hasattr(config, "kind") else None
        self.skeleton = config.model.kind if self.volumetric else None
        self.captures = 0
        self._entries = {}
        self._pool = None
        model.__dict__.setdefault("_train_steps", weakref.WeakSet()).add(self)     # model.to() / load_state_dict invalidate

    def invalidate(self):
        self._entries.clear()
        self._pool = None

    def __call__(self, images_batch, keypoints_3d_gt, keypoints_3d_validity_gt, proj_matricies_batch, batch):
        from .triangulation import _upload, backbone_map_size
        m = self.model
        if not images_batch.is_cuda:
            raise RuntimeError("TrainStep runs on CUDA tensors (got %s)" % images_batch.device)
        if images_batch.shape[1] == 1 and self.base_joint is None:
            raise ValueError("a 1-view batch needs config.kind 'human36m' or 'coco' for its base joint")
        dev = images_batch.device
        cuboids = None
        if self.volumetric:
            B, H, W = images_batch.shape[0], images_batch.shape[3], images_batch.shape[4]
            proj, base, position, step, rots, cuboids = m._host_geometry(batch, B, (H, W), (backbone_map_size(H), backbone_map_size(W)))
            host = _upload(dev, proj, position, base, step, rots)
        else:
            host = (proj_matricies_batch,)
        inputs = (images_batch, keypoints_3d_gt, keypoints_3d_validity_gt) + tuple(host)
        key = self._key(inputs)
        entry = self._entries.get(key)
        if entry is None:
            self._entries = {k: e for k, e in self._entries.items() if k[0][0] != key[0][0]}
            entry = self._capture(inputs)
            self.captures += 1
            self._entries[self._key(inputs)] = entry        # the capture created an empty optimizer state
        for dst, src in zip(entry.static_in, inputs):
            dst.copy_(src)
        m._invalidate_native_eval()             # the replayed Adam and BatchNorm updates bump no tensor version
        entry.graph.replay()
        for p, g in entry.grads:
            p.grad = g
        clone = (lambda t: t.clone()) if self.clone_outputs else (lambda t: t)
        outs = [None if o is None else clone(o) for o in entry.outs]
        metrics = {k: clone(v) for k, v in entry.metrics.items()}
        if self.volumetric:
            kp, features, volumes, vol_conf, coord, base_points = outs
            return (kp, features, volumes, vol_conf, cuboids, coord, base_points), metrics
        return tuple(outs), metrics

    def _key(self, inputs):
        opt = self.optimizer
        groups = tuple(tuple((k, _hashable(v)) for k, v in sorted(g.items()) if k != "params") + (tuple(p.data_ptr() for p in g["params"]),)
                       for g in opt.param_groups)
        state = tuple(v.data_ptr() for g in opt.param_groups for p in g["params"] for v in opt.state.get(p, {}).values()
                      if torch.is_tensor(v))
        return (_model_key(self.model, inputs), groups, state)

    def _capture(self, inputs):
        m, opt = self.model, self.optimizer
        e = _StepEntry()
        e.static_in = [t.detach().clone() for t in inputs]
        params = list(m.parameters())
        opt_params = [p for g in opt.param_groups for p in g["params"]]
        fresh = [p for p in opt_params if not opt.state.get(p)]
        state = [p.detach() for p in params] + _norm_state(m) + [v for p in opt_params for v in opt.state.get(p, {}).values()
                                                                 if torch.is_tensor(v)]

        def drop_grads():
            for p in params + opt_params:
                p.grad = None

        def warm_up():
            drop_grads()
            with warnings.catch_warnings():
                warnings.filterwarnings("ignore", message=".*capturable=True.*")    # "step() is running without CUDA graph capture"
                self._device_step(*e.static_in)
            drop_grads()

        def capture(graph):
            e.graph = torch.cuda.CUDAGraph()
            with graph(e.graph):
                outs, metrics = self._device_step(*e.static_in)
            e.outs = [None if o is None else o.detach() for o in outs]
            e.metrics = {k: v.detach() for k, v in metrics.items()}
            e.grads = [(p, p.grad) for p in params if p.grad is not None]

        def reset():
            for p in fresh:
                for v in opt.state.get(p, {}).values():
                    if torch.is_tensor(v):
                        v.zero_()

        with torch.enable_grad():
            _capture_on_side_stream(self, inputs[0].device, state, warm_up, capture, "TrainStep", reset)
        e.keep = _captured_scratch()
        return e

    def _device_step(self, images, keypoints_gt, validity, *geometry):
        """The captured step: -> (the model's device outputs, metrics)."""
        from . import loss
        m, s = self.model, self.scale
        if self.volumetric:
            kp, features, volumes, vol_conf, coord = m._device_forward(images, *geometry)
            outs = (kp, features, volumes, vol_conf, coord, geometry[2])
        else:
            outs = m._forward_torch(images, geometry[0])
            kp = outs[0]
        valid = (validity > 0.0).float()
        pred, gt = kp, keypoints_gt
        if images.shape[1] == 1:                                   # train.py:200-213, without a boolean-mask index
            rest = (torch.arange(kp.shape[1], device=kp.device) != self.base_joint).view(1, -1, 1)
            j = self.base_joint
            pred = torch.where(rest, kp - kp[:, j:j + 1], kp)
            gt = torch.where(rest, gt - gt[:, j:j + 1], gt)
        crit = loss.keypoints_loss(self.kind, pred * s, gt * s, valid, self.threshold, backend="native")
        metrics = {self.criterion: crit}
        total = crit
        if self.use_ce:
            ce = loss.volumetric_ce_loss(outs[4], outs[2], gt, valid, backend="native")
            metrics["volumetric_ce_loss"] = ce
            total = total + self.ce_weight * ce
        metrics["total_loss"] = total
        torch.autograd.backward(total)
        if self.grad_clip is not None:
            torch.nn.utils.clip_grad_norm_(m.parameters(), self.grad_clip / self.lr)
        grads = [p.grad for p in m.parameters() if p.requires_grad and p.grad is not None]
        norms = torch.stack(torch._foreach_norm(grads)).double()
        metrics["grad_norm_times_lr"] = self.lr * norms.square().sum().sqrt()
        self.optimizer.step()
        with torch.no_grad():
            metrics["l2"] = loss.keypoints_loss("l2", pred.detach() * s, gt * s, valid, backend="native")
            if self.volumetric:
                base_gt = (gt[:, 11, :3] + gt[:, 12, :3]) / 2 if self.skeleton == "coco" else gt[:, 6, :3]
                metrics["base_point_l2"] = torch.sqrt(torch.sum((geometry[2] * s - base_gt * s) ** 2, dim=1)).mean()
        return outs, metrics
