"""lt_b200.TrainStep without a GPU: the constructor's argument checks, the call-time checks, and the metric keys of the step's
device function (run eagerly on the CPU with the torch formulations in place of the kernels)."""
import pytest
import torch

import lt_b200
from lt_b200 import loss as crit, testing


def _vol_config(**opt):
    opt = dict(dict(use_volumetric_ce_loss=True, volumetric_ce_loss_weight=0.01, scale_keypoints_3d=0.1), **opt)
    return testing.make_train_config(testing.make_config(num_layers=18, volume_size=32), criterion="MAE", **opt)


def _alg_config(**opt):
    opt = dict(dict(mse_smooth_threshold=400, scale_keypoints_3d=0.1), **opt)
    return testing.make_train_config(testing.make_alg_config(num_layers=18), criterion="MSESmooth", **opt)


def _vol(cfg, backend="hybrid"):
    return lt_b200.VolumetricTriangulationNet(cfg, device="cpu", backend=backend)


def _alg(cfg, backend="hybrid"):
    return lt_b200.AlgebraicTriangulationNet(cfg, device="cpu", backend=backend)


def _adam(m, **kw):
    return torch.optim.Adam(m.parameters(), lr=1e-4, **dict(dict(capturable=True), **kw))


@pytest.mark.parametrize("make, config", [(_vol, _vol_config), (_alg, _alg_config)])
def test_argument_checks(make, config):
    cfg = config()
    m = make(cfg)
    lt_b200.TrainStep(m, _adam(m), cfg)
    with pytest.raises(ValueError, match="hybrid"):
        t = make(config(), backend="torch")
        lt_b200.TrainStep(t, _adam(t), cfg)
    with pytest.raises(ValueError, match="capturable=True"):
        lt_b200.TrainStep(m, _adam(m, capturable=False), cfg)
    with pytest.raises(ValueError, match="capturable=True"):
        lt_b200.TrainStep(m, torch.optim.SGD(m.parameters(), lr=1e-3), cfg)
    opt = _adam(m)
    opt.param_groups[0]["capturable"] = False
    with pytest.raises(ValueError, match="capturable=True"):
        lt_b200.TrainStep(m, opt, cfg)
    bad = config()
    bad.opt.criterion = "Huber"
    with pytest.raises(ValueError, match="criterion"):
        lt_b200.TrainStep(m, _adam(m), bad)
    bad = config()
    bad.model.name = "alg" if make is _vol else "vol"
    with pytest.raises(ValueError, match="config.model.name"):
        lt_b200.TrainStep(m, _adam(m), bad)
    with pytest.raises(ValueError, match="AlgebraicTriangulationNet or a VolumetricTriangulationNet"):
        lt_b200.TrainStep(m.backbone, _adam(m), cfg)
    r = lt_b200.RANSACTriangulationNet(testing.make_ransac_config(num_layers=18), device="cpu", backend="torch")
    with pytest.raises(ValueError, match="AlgebraicTriangulationNet or a VolumetricTriangulationNet"):
        lt_b200.TrainStep(r, _adam(m), cfg)


def test_distributed_data_parallel_is_refused():
    cfg = _alg_config()
    m = _alg(cfg)
    ddp = torch.nn.parallel.DistributedDataParallel.__new__(torch.nn.parallel.DistributedDataParallel)
    torch.nn.Module.__init__(ddp)
    ddp.module = m
    with pytest.raises(ValueError, match="DistributedDataParallel"):
        lt_b200.TrainStep(ddp, _adam(m), cfg)


def test_config_combinations_the_reference_cannot_run_are_refused():
    cfg = _alg_config(use_volumetric_ce_loss=True)
    m = _alg(cfg)
    with pytest.raises(ValueError, match="volumetric model"):
        lt_b200.TrainStep(m, _adam(m), cfg)
    cfg = _vol_config()
    cfg.model.kind = "h36m"
    m = _vol(cfg)
    with pytest.raises(ValueError, match="model.kind"):
        lt_b200.TrainStep(m, _adam(m), cfg)


def test_call_time_checks():
    cfg = _alg_config()
    cfg.kind = "cmu"
    m = _alg(cfg)
    step = lt_b200.TrainStep(m, _adam(m), cfg)
    images, batch = testing.make_batch(2, 1, image_size=64)
    with pytest.raises(RuntimeError, match="CUDA"):
        step(*testing.prepare_batch(batch, images, "cpu"), batch)
    fake = torch.zeros(2, 1, 3, 64, 64)          # the kind check comes before any device work: a tensor that reports CUDA
    fake.__class__ = type("FakeCuda", (torch.Tensor,), {"is_cuda": property(lambda self: True)})
    with pytest.raises(ValueError, match="1-view batch"):
        step(fake, None, None, None, batch)


@pytest.mark.parametrize("make, config, keys", [
    (_vol, _vol_config, {"MAE", "volumetric_ce_loss", "total_loss", "grad_norm_times_lr", "l2", "base_point_l2"}),
    (_alg, _alg_config, {"MSESmooth", "total_loss", "grad_norm_times_lr", "l2"}),
])
def test_metric_keys_follow_train_py(make, config, keys, monkeypatch):
    """The captured function itself, eagerly on the CPU: torch formulations for the kernels, a plain Adam for the capturable one."""
    cfg = config(grad_clip=1e-4)
    m = make(cfg)
    step = lt_b200.TrainStep(m, _adam(m), cfg)
    m.backend = "torch"
    step.optimizer = torch.optim.Adam(m.parameters(), lr=1e-4)
    monkeypatch.setattr(crit, "_resolve_backend", lambda backend, *t: "torch")
    S = 64 if make is _vol else 128                              # the confidence head pools the algebraic model's features to 1x1
    images, batch = testing.make_batch(2, 2, image_size=S)
    images, kp, valid, proj = testing.prepare_batch(batch, images, "cpu")
    m.train()
    if make is _vol:
        from lt_b200.triangulation import _upload
        geometry = _upload(torch.device("cpu"), *m._host_geometry(batch, 2, (64, 64), (16, 16))[:5])
        outs, metrics = step._device_step(images, kp, valid, *geometry)
        assert len(outs) == 6
    else:
        outs, metrics = step._device_step(images, kp, valid, proj)
        assert len(outs) == 4
    assert set(metrics) == keys
    assert all(v.dim() == 0 and bool(torch.isfinite(v)) for v in metrics.values())
    assert all(p.grad is not None for p in m.parameters() if p.requires_grad)
    norm = sum(float(p.grad.norm()) ** 2 for p in m.parameters() if p.requires_grad) ** 0.5       # misc.calc_gradient_norm
    assert abs(float(metrics["grad_norm_times_lr"]) - 1e-4 * norm) <= 1e-6 * 1e-4 * norm
    assert norm <= (1e-4 / 1e-4) * (1 + 1e-5)                  # clipped to grad_clip / lr = 1
