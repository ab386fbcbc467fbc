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
        key = (tuple((tuple(t.shape), t.dtype, t.device) for t in inputs), tuple(p.requires_grad for p in params),
               tuple(p.data_ptr() for p in params), tuple(b.data_ptr() for b in model.buffers()),
               tuple(m.training for m in model.modules()))
        entry = self._entries.get(key)
        if entry is None:
            entry = self._entries[key] = self._capture(model, fn, inputs, params)
            self.captures += 1
        for dst, src in zip(entry.static_in, inputs):
            dst.copy_(src)
        outs = iter(_Replay.apply(self, entry, clone_outputs, *entry.params))
        return tuple(next(outs) if present else None for present in entry.layout)

    def _capture(self, model, fn, inputs, params):
        dev = inputs[0].device
        e = _Entry()
        e.params = [p for p in params if p.requires_grad]
        e.static_in = [t.detach().clone() for t in inputs]
        state = _norm_state(model)
        saved = [b.clone() for b in state]
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(cur)
        try:
            with torch.cuda.device(dev), torch.autograd.set_detect_anomaly(False), torch.cuda.stream(side):
                outs = fn(*e.static_in)
                diff = [o for o in outs if o is not None and o.requires_grad]
                torch.autograd.grad(diff, e.params, [torch.zeros_like(o) for o in diff], allow_unused=True)
                del outs, diff
                if self._pool is None:
                    self._pool = torch.cuda.graph_pool_handle()
                e.fwd, e.bwd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                with torch.cuda.graph(e.fwd, pool=self._pool, stream=side, capture_error_mode="thread_local"):
                    outs = fn(*e.static_in)
                present = [o for o in outs if o is not None]
                e.diff = [o.requires_grad for o in present]
                diff = [o for o in present if o.requires_grad]
                e.gouts = [torch.zeros_like(o) for o in diff]
                e.gout_zero = [True] * len(diff)
                with torch.cuda.graph(e.bwd, pool=self._pool, stream=side, capture_error_mode="thread_local"):
                    grads = torch.autograd.grad(diff, e.params, e.gouts, allow_unused=True)
                    used = [g.reshape(-1) for g in grads if g is not None]
                    e.flat = torch.cat(used) if used else None
                e.grad_shapes = [None if g is None else g.shape for g in grads]
                e.outs = [o.detach() for o in present]
                e.layout = [o is not None for o in outs]
                del outs, present, diff, grads, used
        except Exception as exc:
            raise RuntimeError("train_graph: capturing the training step failed: %s: %s" % (type(exc).__name__, exc)) from exc
        finally:
            cur.wait_stream(side)
            with torch.cuda.stream(cur):
                for b, s in zip(state, saved):
                    b.copy_(s)
        # scratch the captured launches write at fixed addresses: an eager call that grows a workspace later must not free it
        e.keep = list(autograd_ops._WORKSPACE.values()) + list(engine._SPLITK_WS.values())
        return e
