"""Synthetic workload factory shared by tests, bench.py and __graft_entry__.smoke().

Nothing here is on the product path: it builds the experiment config (same schema as
experiments/human36m/*/human36m_vol_softmax.yaml), a ring of pinhole cameras, the `batch` dict in
the collate layout (mvn/datasets/utils.py:8-37) and a seeded, well-conditioned weight set.
(SURVEY.md section 8d defines the rig; Human3.6M and the released weights are not obtainable offline.)
"""
import numpy as np
import torch
from torch import nn

from .multiview import Camera


class AttrDict(dict):
    """10-line EasyDict stand-in: attribute access, AttributeError for missing keys (hasattr probes work)."""

    def __init__(self, d=None, **kw):
        super().__init__()
        for k, v in dict(d or {}, **kw).items():
            self[k] = AttrDict(v) if isinstance(v, dict) else v

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v


def make_config(num_layers=152, volume_size=64, aggregation="softmax", volume_multiplier=1.0, volume_softmax=True,
                use_gt_pelvis=True, kind="mpii", cuboid_side=2500.0, num_joints=17, style="simple"):
    """The `model:` section of human36m_vol_softmax.yaml with init_weights off (random init, BASELINE.json)."""
    return AttrDict({
        "image_shape": [384, 384],
        "model": {
            "name": "vol", "kind": kind, "volume_aggregation_method": aggregation,
            "init_weights": False, "use_gt_pelvis": use_gt_pelvis, "cuboid_side": cuboid_side,
            "volume_size": volume_size, "volume_multiplier": volume_multiplier, "volume_softmax": volume_softmax,
            "heatmap_softmax": True, "heatmap_multiplier": 100.0,
            "backbone": {"name": "resnet%d" % num_layers, "style": style, "init_weights": False,
                         "num_joints": num_joints, "num_layers": num_layers},
        },
    })


def _look_at(eye, target=(0.0, 0.0, 900.0)):
    """World->camera rotation for a camera at `eye` looking at `target`, z up (H3.6M-like, mm)."""
    eye, target = np.asarray(eye, dtype=np.float64), np.asarray(target, dtype=np.float64)
    fwd = target - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, np.array([0.0, 0.0, 1.0]))
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    return np.stack([right, down, fwd], axis=0)


def make_cameras(n_views, image_size=384, radius=4500.0, height=1500.0, focal=None, phase=0.3, camera_cls=Camera):
    """n_views pinhole cameras on a ring looking at the subject; the 2.5 m cuboid fills the crop."""
    focal = focal if focal is not None else 520.0 * image_size / 384.0
    cams = []
    for v in range(n_views):
        a = phase + 2 * np.pi * v / n_views
        eye = np.array([radius * np.cos(a), radius * np.sin(a), height])
        R = _look_at(eye)
        t = -R @ eye
        K = np.array([[focal, 0.0, image_size / 2.0], [0.0, focal, image_size / 2.0], [0.0, 0.0, 1.0]])
        cams.append(camera_cls(R, t, K, name="cam%d" % v))
    return cams


def make_batch(batch_size, n_views, image_size=384, seed=0, camera_cls=Camera, device="cpu"):
    """-> images (B, V, 3, H, W) float32, batch dict with cameras[v][b], keypoints_3d, pred_keypoints_3d."""
    rng = np.random.RandomState(seed)
    g = torch.Generator().manual_seed(seed)
    images = torch.randn(batch_size, n_views, 3, image_size, image_size, generator=g)
    cams = make_cameras(n_views, image_size, camera_cls=camera_cls)
    cameras = [[camera_cls(c.R, c.t, c.K, name=c.name) for _ in range(batch_size)] for c in cams]
    kps = []
    for _ in range(batch_size):
        kp = np.concatenate([rng.normal(0.0, 200.0, size=(17, 3)) + np.array([0.0, 0.0, 900.0]), np.ones((17, 1))], axis=1)
        kps.append(kp)
    batch = {"cameras": cameras, "keypoints_3d": kps,
             "pred_keypoints_3d": np.stack([k[:, :3] for k in kps], axis=0)}
    return images.to(device), batch


@torch.no_grad()
def randomize_weights(model, seed=0, calib_size=64, calib_views=2, feat_gain=4.0, branch_gain=0.2):
    """Seeded, non-degenerate weights (SURVEY.md hard part H1).

    Default inits in eval mode collapse the signal (BN running stats are 0/1, deconv outputs ~5e-3),
    which would make any parity check vacuous.  Recipe: Kaiming-normal conv filters, BatchNorm running
    affine gamma ~ U(0.75, 1.25), beta ~ N(0, 0.2), then running statistics calibrated by one train-mode
    pass of the torch formulation over seeded noise (momentum 1) and the output layer rescaled.  Deterministic for a given torch build.
    """
    g = torch.Generator().manual_seed(seed)
    dev = next(model.parameters()).device
    model_cpu = model.to("cpu")
    for mod in model_cpu.modules():
        if isinstance(mod, (nn.Conv2d, nn.Conv3d, nn.ConvTranspose2d, nn.ConvTranspose3d)):
            fan_in = mod.weight[0].numel() if not isinstance(mod, (nn.ConvTranspose2d, nn.ConvTranspose3d)) \
                else mod.weight.shape[0] * mod.weight[0, 0].numel() / (mod.stride[0] ** (mod.weight.dim() - 2))
            mod.weight.copy_(torch.randn(mod.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
            if mod.bias is not None:
                mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.05)
    bns = [m for m in model_cpu.modules() if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm3d))]
    saved = [(m.momentum, m.training) for m in bns]
    # last BatchNorm of every residual branch: small gain, so that the identity path dominates (as in trained
    # residual nets; a random ResNet with unit-gain branches amplifies a 1e-5 perturbation ~250x, which would turn
    # the parity check into a test of fp32 summation order)
    last_of_branch = set()
    for mod in model_cpu.modules():
        if hasattr(mod, "stages") and hasattr(mod, "downsample"):
            last_of_branch.add(mod.stages()[-1][1])
        if hasattr(mod, "res_branch"):
            last_of_branch.add(mod.res_branch[4])
    for m in bns:
        # affine parameters first, so that the calibration below sees the final network
        lo, hi = (branch_gain * 0.5, branch_gain * 1.5) if m in last_of_branch else (0.75, 1.25)
        m.weight.copy_(torch.rand(m.weight.shape, generator=g) * (hi - lo) + lo)
        m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.2)
        m.momentum = 1.0
        m.train()
    # calibration pass: the whole torch formulation (backbone -> process_features -> unprojection -> V2V) on a
    # synthetic scene, so every BatchNorm sees the activation statistics it will see at test time
    model_cpu.process_features[0].weight.mul_(feat_gain)   # wider feature range: view-softmax becomes selective
    # enough samples that the deepest V2V level (1^3 voxels per sample at volume_size 32) has stable statistics
    calib_batch = 2 if model_cpu.volume_size >= 64 else 6
    images, batch = make_batch(calib_batch, calib_views, image_size=calib_size, seed=seed + 1000)
    grabbed = {}
    hook = model_cpu.volume_net.output_layer.register_forward_hook(lambda m, i, o: grabbed.update(logits=o))
    top_training = model_cpu.training
    model_cpu.training = False                               # theta = 0; only the BatchNorms are in train mode
    backend, model_cpu.backend = getattr(model_cpu, "backend", "torch"), "torch"    # CPU calibration: torch ops whatever the backend
    model_cpu._forward_torch(images, batch)
    model_cpu.backend = backend
    model_cpu.training = top_training
    hook.remove()
    logits = grabbed["logits"]
    for m, (mom, tr) in zip(bns, saved):
        m.momentum = mom
        m.train(tr)
        m.running_var.clamp_(min=1e-3)
    # logits with a spread of ~2.5: the 3-D softmax is peaked but not saturated
    model_cpu.volume_net.output_layer.weight.mul_(2.5 / float(logits.std()))
    model_cpu.eval()
    return model_cpu.to(dev)


def make_alg_config(num_layers=152, use_confidences=True, heatmap_multiplier=100.0, num_joints=17):
    """The `model:` section of experiments/human36m/*/human36m_alg.yaml with init_weights off."""
    return AttrDict({
        "image_shape": [384, 384],
        "model": {"name": "alg", "init_weights": False, "use_confidences": use_confidences,
                  "heatmap_multiplier": heatmap_multiplier, "heatmap_softmax": True,
                  "backbone": {"name": "resnet%d" % num_layers, "style": "simple", "init_weights": False,
                               "num_joints": num_joints, "num_layers": num_layers}},
    })


def image_projections(batch):
    """(B, V, 3, 4) float32 image-space projection matrices of a make_batch() dict (datasets/utils.py:61-63)."""
    from .multiview import stack_projections
    return stack_projections(batch["cameras"])


@torch.no_grad()
def randomize_backbone_weights(model, seed=0, calib_size=128, calib_images=4, branch_gain=0.2, heat_spread=3.0):
    """Seeded well-conditioned weights for a model that only has `.backbone` (algebraic model): same recipe as
    randomize_weights; the heatmap head is rescaled so that heatmaps * heatmap_multiplier has a spread of ~3."""
    g = torch.Generator().manual_seed(seed)
    dev = next(model.parameters()).device
    m = model.to("cpu")
    bb = m.backbone
    for mod in bb.modules():
        if isinstance(mod, (nn.Conv2d, nn.ConvTranspose2d)):
            fan_in = mod.weight[0].numel() if isinstance(mod, nn.Conv2d) else mod.weight.shape[0] * mod.weight[0, 0].numel() / 4
            mod.weight.copy_(torch.randn(mod.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
            if mod.bias is not None:
                mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.05)
        if isinstance(mod, nn.Linear):
            mod.weight.copy_(torch.randn(mod.weight.shape, generator=g) * (1.0 / mod.weight.shape[1]) ** 0.5)
            mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.3)
    last = {u.stages()[-1][1] for u in bb.modules() if hasattr(u, "stages")}
    bns = [x for x in bb.modules() if isinstance(x, nn.BatchNorm2d)]
    for x in bns:
        lo, hi = (branch_gain * 0.5, branch_gain * 1.5) if x in last else (0.75, 1.25)
        x.weight.copy_(torch.rand(x.weight.shape, generator=g) * (hi - lo) + lo)
        x.bias.copy_(torch.randn(x.bias.shape, generator=g) * 0.2)
        x.momentum = 1.0
        x.train()
    heat, _, _, _ = bb(torch.randn(calib_images, 3, calib_size, calib_size, generator=g))
    for x in bns:
        x.momentum = BN_MOMENTUM
        x.eval()
        x.running_var.clamp_(min=1e-3)
    scale = heat_spread / (float(heat.std()) * float(m.heatmap_multiplier))
    bb.final_layer.weight.mul_(scale)
    bb.final_layer.bias.mul_(scale)
    m.eval()
    return m.to(dev)


BN_MOMENTUM = 0.1


def make_ransac_config(num_layers=152, direct_optimization=True, num_joints=17):
    """The `model:` section of experiments/human36m/eval/human36m_ransac.yaml with init_weights off."""
    return AttrDict({
        "image_shape": [384, 384],
        "model": {"name": "ransac", "init_weights": False, "direct_optimization": direct_optimization,
                  "backbone": {"name": "resnet%d" % num_layers, "style": "simple", "init_weights": False,
                               "num_joints": num_joints, "num_layers": num_layers}},
    })


class _BackboneHolder(nn.Module):
    def __init__(self, backbone):
        super().__init__()
        self.backbone = backbone
        self.heatmap_multiplier = 1.0


@torch.no_grad()
def randomize_ransac_weights(model, seed=0, calib_size=64):
    """randomize_backbone_weights for a model whose heat maps are used raw (RANSACTriangulationNet): heat-map spread ~3."""
    randomize_backbone_weights(_BackboneHolder(model.backbone), seed=seed, calib_size=calib_size)
    return model.eval()


# ---- restated training loop of the reference (train.py:185-263), for the TrainStep tests and tools/train_step_timing.py ----------

CRITERIA = {"MSE": "mse", "MSESmooth": "mse_smooth", "MAE": "mae"}


def reference_keypoints_loss(kind, pred, gt, validity, threshold=400):
    """Restatement of the reference's keypoint criteria (mvn/models/loss.py:7-49), `kind` one of "mse", "mse_smooth", "mae", "l2":
    the divisor read to the host with .item() and MSESmooth's boolean-mask replacement, as there.  Runs in the inputs' dtype
    (float64 inputs give the float64 reference of the tests)."""
    divisor = max(1, torch.sum(validity).item())
    if kind == "l2":
        return torch.sum(torch.sqrt(torch.sum((gt - pred) ** 2 * validity, dim=2))) / divisor
    if kind == "mae":
        terms = torch.abs(gt - pred) * validity
    else:
        terms = (gt - pred) ** 2 * validity
        if kind == "mse_smooth":
            over = terms > threshold
            terms[over] = torch.pow(terms[over], 0.1) * (threshold ** 0.9)
    return torch.sum(terms) / (pred.shape[-1] * divisor)


def make_train_config(model_config, criterion="MAE", lr=1e-4, kind="human36m", **opt):
    """A train.py config: `model_config` (make_config / make_alg_config) with a top-level `kind` and an `opt` section."""
    cfg = AttrDict(model_config)
    cfg.kind = kind
    cfg.opt = AttrDict(dict(criterion=criterion, lr=lr, **opt))
    return cfg


def recipe_optimizer(model, config, **adam):
    """train.py:428-439's Adam: per-module lrs for the volumetric model, the trainable parameters for the algebraic one."""
    o = config.opt
    if config.model.name == "vol":
        groups = [{"params": model.backbone.parameters()},
                  {"params": model.process_features.parameters(), "lr": getattr(o, "process_features_lr", o.lr)},
                  {"params": model.volume_net.parameters(), "lr": getattr(o, "volume_net_lr", o.lr)}]
        return torch.optim.Adam(groups, lr=o.lr, **adam)
    return torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=o.lr, **adam)


def reference_train_step(model, optimizer, config, images_batch, keypoints_3d_gt, keypoints_3d_validity_gt, proj_matricies_batch,
                         batch):
    """One eager iteration of the reference's training loop body (train.py:185-263) restated: the model, the restated criterion,
    lt_b200's native VolumetricCELoss, every .item() of the loop, the per-parameter .item() gradient norm of misc.calc_gradient_norm,
    clip_grad_norm_ and the optimizer step.  base_point_l2 takes coco's hip midpoint from the ground truth.
    -> (the model's outputs, metric_dict of Python floats)."""
    from .loss import VolumetricCELoss
    o = config.opt
    outputs = model(images_batch, proj_matricies_batch, batch)
    kp, gt = outputs[0], keypoints_3d_gt
    J = kp.shape[1]
    valid = (keypoints_3d_validity_gt > 0.0).type(torch.float32)
    s = o.scale_keypoints_3d if hasattr(o, "scale_keypoints_3d") else 1.0
    if images_batch.shape[1] == 1:
        base_joint = {"human36m": 6, "coco": 11}[config.kind]
        gt = gt.clone()
        gt[:, torch.arange(J) != base_joint] -= gt[:, base_joint:base_joint + 1]
        kp = kp.clone()
        kp[:, torch.arange(J) != base_joint] -= kp[:, base_joint:base_joint + 1]
    metrics = {}
    threshold = o.mse_smooth_threshold if o.criterion == "MSESmooth" else 400
    loss = reference_keypoints_loss(CRITERIA[o.criterion], kp * s, gt * s, valid, threshold)
    total = 0.0 + loss
    metrics[o.criterion] = loss.item()
    if getattr(o, "use_volumetric_ce_loss", False):
        ce = VolumetricCELoss(backend="native")(outputs[5], outputs[2], gt, valid)
        metrics["volumetric_ce_loss"] = ce.item()
        total = total + getattr(o, "volumetric_ce_loss_weight", 1.0) * ce
    metrics["total_loss"] = total.item()
    optimizer.zero_grad()
    total.backward()
    if hasattr(o, "grad_clip"):
        torch.nn.utils.clip_grad_norm_(model.parameters(), o.grad_clip / o.lr)
    norm2 = 0.0
    for p in model.parameters():
        if p.requires_grad:
            norm2 += p.grad.data.norm(2).item() ** 2
    metrics["grad_norm_times_lr"] = o.lr * norm2 ** 0.5
    optimizer.step()
    metrics["l2"] = reference_keypoints_loss("l2", kp * s, gt * s, valid).item()
    if config.model.name == "vol":
        base_pred = outputs[6]
        per = []
        for b in range(kp.shape[0]):
            base_gt = (gt[b, 11, :3] + gt[b, 12, :3]) / 2 if config.model.kind == "coco" else gt[b, 6, :3]
            per.append(torch.sqrt(torch.sum((base_pred[b] * s - base_gt * s) ** 2)).item())
        metrics["base_point_l2"] = float(np.mean(per))
    return outputs, metrics


def prepare_batch(batch, images, device):
    """images, keypoints_3d (B, J, 3), validity (B, J, 1), image-space projections as the reference's prepare_batch returns them
    (datasets/utils.py:41-66) for a make_batch() dict."""
    kp = torch.from_numpy(np.stack(batch["keypoints_3d"])).float()
    return (images.to(device), kp[..., :3].to(device), kp[..., 3:].to(device),
            torch.from_numpy(image_projections(batch)).to(device))


def keypoint_case(name, dim=3, n=(3, 5), seed=0):
    """(pred, gt, validity (B, J, 1)) float32 of one graded case of the keypoint criteria tests (KEYPOINT_CASES)."""
    g = torch.Generator().manual_seed(seed)
    B, J = n
    gt = torch.randn(B, J, dim, generator=g) * 30
    pred = gt + torch.randn(B, J, dim, generator=g) * 15
    v = (torch.rand(B, J, 1, generator=g) > 0.3).float()
    if name == "zero_validity":
        v.zero_()
    elif name == "fractional":
        v = torch.rand(B, J, 1, generator=g)
    elif name == "boundary":                    # (gt - pred)^2 v = 400 exactly, and just above it
        v[0, 0], v[0, 1] = 1.0, 1.0
        pred[0, 0, 0] = gt[0, 0, 0] - 20.0
        pred[0, 1, 0] = gt[0, 1, 0] - 20.0009765625
    elif name == "nan_invalid":
        v[1, 2] = 0.0
        pred[1, 2, 0] = float("nan")
        v[0, 3] = 0.0
        pred[0, 3, 1] = float("inf")
    elif name == "nan_valid":
        v[1, 1] = 1.0
        pred[1, 1, 0] = float("nan")
    elif name == "many":                        # more points than the CTA's threads
        return keypoint_case("plain", dim, (20, 17), seed)
    return pred, gt, v


KEYPOINT_CASES = ("plain", "zero_validity", "fractional", "boundary", "nan_invalid", "nan_valid", "many")


def reference_keypoints_loss64(kind, pred, gt, v, threshold=400.0):
    """float64 loss, gradient wrt pred (grad_loss 1) and sum of |terms| of the restated reference."""
    p = pred.double().requires_grad_(True)
    loss = reference_keypoints_loss(kind, p, gt.double(), v.double(), threshold)
    loss.backward()
    with torch.no_grad():
        r = gt.double() - pred.double()
        terms = torch.abs(r) * v if kind == "mae" else r ** 2 * v.double()
        if kind == "l2":
            terms = torch.sqrt(terms.sum(-1))
    return float(loss.detach()), p.grad, float(terms.abs().nansum())
