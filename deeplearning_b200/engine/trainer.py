"""Data-parallel training step: flat parameter / gradient arenas, ONE gradient all-reduce, one fused optimizer launch.

H100-native counterpart of the reference's DDP recipe (others/train_with_DDP/train.py:106-111,188-201,245-253 and
classification/swin_transformer/main.py:101-103): one process per GPU, identical replicas, per-GPU BatchNorm statistics
(DDP *without* SyncBN, as the north-star asks), gradients averaged across ranks after backward, identical update on every
rank.  The backward kernels write straight into one contiguous fp32 arena; like DDP's bucketed reducer the all-reduce is
overlapped with the backward pass: gradients are produced from the end of the arena towards its start, and every time a
stretch of ``bucket_mb`` of completed gradients has accumulated it is all-reduced (NCCL over NVLink/NVSwitch) on a side
stream while the remaining layers are still computing.  The 1/world scale is folded into the fused optimizer kernel, and
the whole step (collectives included) is captured in ONE CUDA graph.

``model.parameters()`` keep their identity: each ``p.data`` becomes a view into the parameter arena and ``p.grad`` a
view into the gradient arena, so ``state_dict()`` / checkpoints / user code reading ``.grad`` behave as in the reference.
"""
import os

import torch
import torch.distributed as dist

from .. import ops
from .common import padded_classes
from .packing import weight_cache


def _engine_for(model):
    from ..classification.resnet.models.networks import ResNet

    if isinstance(model, ResNet):
        from . import resnet

        return resnet
    from ..classification.vision_transformer.vit_model import VisionTransformer

    if isinstance(model, VisionTransformer):
        from . import vit

        return vit
    from ..classification.convNext.models.networks import ConvNeXt

    if isinstance(model, ConvNeXt):
        from . import convnext

        return convnext
    from ..classification.swin_transformer.models.swin_transformer import SwinTransformer

    if isinstance(model, SwinTransformer):
        from . import swin

        return swin
    from ..classification.RepVGG.models.repvgg import RepVGG

    if isinstance(model, RepVGG):
        from . import repvgg

        return repvgg
    from ..classification.efficientNet.models.network import EfficientNet

    if isinstance(model, EfficientNet):
        from . import efficientnet

        return efficientnet
    from ..classification.vggNet.models.network import VGG

    if isinstance(model, VGG):
        from . import vgg

        return vgg
    raise NotImplementedError(f"no GPU engine schedule for {type(model).__name__}")


def ops_clip_blocks():
    from .. import _lib

    return _lib.load().b200_grad_clip_blocks()


class FlatArena:
    """Parameters, gradients and optimizer state of a model as three contiguous fp32 buffers (device agnostic host logic).

    Every ``p.data`` becomes a view into ``flat_p`` and every ``p.grad`` a view into ``flat_g``; ``all_reduce_grads`` is the
    single collective of the data-parallel step and ``broadcast`` makes the replicas identical at start-up."""

    def __init__(self, params, process_group=None, world_size=None, bucket_mb=25.0):
        self.params = [p for p in params if p.requires_grad]
        self.bucket_elems = max(1, int(bucket_mb * 1e6 / 4))
        self._comm = None
        if not self.params:
            raise ValueError("no trainable parameters")
        self.group = process_group
        if world_size is None:
            world_size = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
        self.world = world_size
        dev = self.params[0].device
        self.offsets, total = [], 0
        for p in self.params:
            if p.device != dev or p.dtype != torch.float32:
                raise ValueError("all parameters must be fp32 tensors on one device")
            self.offsets.append(total)
            total += (p.numel() + 3) // 4 * 4  # keep every slot 16-byte aligned
        self.flat_p = torch.zeros(total, dtype=torch.float32, device=dev)
        self.flat_g = torch.zeros(total, dtype=torch.float32, device=dev)
        self.flat_m = torch.zeros(total, dtype=torch.float32, device=dev)
        self._gviews = {}
        with torch.no_grad():
            for p, o in zip(self.params, self.offsets):
                pv = self.flat_p[o:o + p.numel()].view(p.shape)
                pv.copy_(p.data)
                p.data = pv
                gv = self.flat_g[o:o + p.numel()].view(p.shape)
                p.grad = gv
                self._gviews[p.data_ptr()] = gv

    def grad_view(self, param):
        return self._gviews.get(param.data_ptr())

    # ---- overlapped all-reduce: the engines produce gradients roughly in reverse parameter order ------------------------
    def begin_backward(self):
        """Start tracking which gradients are final (``notify``) so that completed stretches [lo, hi) at the END of the
        arena can be all-reduced while the backward pass is still running."""
        self._index = {p.data_ptr(): i for i, p in enumerate(self.params)}
        self._done = [False] * len(self.params)
        self._next = len(self.params) - 1          # highest-offset parameter whose gradient is still outstanding
        self._hi = self.flat_g.numel()             # everything in [_hi, end) has been handed to NCCL already
        self.buckets_launched = 0
        if self._comm is None and self.flat_g.is_cuda:
            self._comm = torch.cuda.Stream()

    def notify(self, param):
        if self.world <= 1 or getattr(self, "_done", None) is None:
            return
        i = self._index.get(param.data_ptr())
        if i is None or self._done[i]:
            return
        self._done[i] = True
        while self._next >= 0 and self._done[self._next]:
            self._next -= 1
        lo = self.offsets[self._next + 1] if self._next + 1 < len(self.offsets) else self.flat_g.numel()
        if self._next < 0:
            lo = 0
        if self._hi - lo >= self.bucket_elems or (lo == 0 and self._hi > 0):
            self._reduce_range(lo, self._hi)
            self._hi = lo

    def _reduce_range(self, lo, hi):
        if hi <= lo:
            return
        chunk = self.flat_g[lo:hi]
        if self._comm is not None:
            ev = torch.cuda.Event()
            ev.record()
            with torch.cuda.stream(self._comm):
                self._comm.wait_event(ev)
                dist.all_reduce(chunk, op=dist.ReduceOp.SUM, group=self.group)
        else:
            dist.all_reduce(chunk, op=dist.ReduceOp.SUM, group=self.group)
        self.buckets_launched += 1

    def finish_backward(self):
        """Reduce whatever has not been handed to NCCL yet and make the compute stream wait for the collectives."""
        if self.world <= 1 or getattr(self, "_done", None) is None:
            self._done = None
            return
        self._reduce_range(0, self._hi)
        self._hi = 0
        self._done = None
        if self._comm is not None:
            torch.cuda.current_stream().wait_stream(self._comm)

    def broadcast(self, buffers=()):
        if self.world > 1:
            dist.broadcast(self.flat_p, src=0, group=self.group)  # identical replicas (train_with_DDP/train.py:171-176)
            for b in buffers:
                dist.broadcast(b, src=0, group=self.group)

    def all_reduce_grads(self):
        """SUM over ranks; the 1/world average is folded into the optimizer kernel (``grad_scale``)."""
        if self.world > 1:
            dist.all_reduce(self.flat_g, op=dist.ReduceOp.SUM, group=self.group)

    @property
    def grad_scale(self):
        return 1.0 / self.world


def no_decay_rule(name, param):
    """Weight-decay grouping of the reference AdamW recipes: 1-D parameters and biases are not decayed
    (classification/convNext/utils.py:144-166 ``get_params_groups``)."""
    return param.dim() == 1 or name.endswith(".bias")


def model_no_decay_rule(model):
    """Decay grouping of the reference Swin recipe (classification/swin_transformer/utils/optimizer.py:41-63
    ``set_weight_decay``): 1-D parameters, biases, names in ``model.no_weight_decay()`` and names containing a keyword of
    ``model.no_weight_decay_keywords()`` are not decayed."""
    skip = set(model.no_weight_decay()) if hasattr(model, "no_weight_decay") else set()
    keywords = tuple(model.no_weight_decay_keywords()) if hasattr(model, "no_weight_decay_keywords") else ()

    def rule(name, param):
        return no_decay_rule(name, param) or name in skip or any(k in name for k in keywords)

    return rule


class _GradSink:
    """Gradient destination handed to the engines: views of the arena, plus completion notices for the overlapped reduce."""

    def __init__(self, arena):
        self.arena = arena

    def __call__(self, param):
        return self.arena.grad_view(param)

    def notify(self, param):
        self.arena.notify(param)


class TrainStep:
    def __init__(self, model, lr=0.01, momentum=0.9, weight_decay=5e-5, process_group=None, world_size=None,
                 broadcast=True, optimizer="sgd", betas=(0.9, 0.999), eps=1e-8, no_decay=None, clip_grad=None,
                 overlap=True, bucket_mb=25.0, label_smoothing=0.0, accum_steps=1):
        """optimizer="sgd": torch.optim.SGD(momentum, weight_decay on every parameter) - resnet/vit train.py:96,94.
        optimizer="adamw": torch.optim.AdamW(betas, eps, weight_decay) with the reference's decay / no-decay groups
        (``no_decay(name, param) -> bool``, default ``no_decay_rule``) - convNext/train.py:96,102.
        optimizer="adam": torch.optim.Adam(lr, betas, eps, weight_decay) in one group, every parameter decayed by an L2 term
        added to the gradient (not AdamW's decoupled decay) - vggNet/train.py:133-136.
        clip_grad: max global L2 norm of the (all-reduced, averaged) gradient, ``clip_grad_norm_`` of the Swin recipe
        (swin_transformer/main.py:197, config TRAIN.CLIP_GRAD = 5.0); the norm of the last step is ``self.grad_norm``.
        label_smoothing: LabelSmoothingCrossEntropy of the Swin recipe (main.py:114-115); floating-point ``labels`` of
        shape [B, num_classes] (Mixup / CutMix targets, engine/mixup.py) select SoftTargetCrossEntropy (main.py:111-113).
        accum_steps: gradient accumulation (main.py:190-199, TRAIN.ACCUMULATION_STEPS): every call runs forward + backward of
        one micro-batch with the loss gradient scaled by 1/accum_steps; the all-reduce, clipping and the optimizer update
        happen on every accum_steps-th call."""
        self.model = model
        self.engine = _engine_for(model)
        self.lr, self.momentum, self.weight_decay = lr, momentum, weight_decay
        self.optimizer, self.betas, self.eps = optimizer, betas, eps
        if optimizer not in ("sgd", "adamw", "adam"):
            raise ValueError(f"unknown optimizer {optimizer!r}")
        bucket_mb = float(os.environ.get("B200_BUCKET_MB", bucket_mb))   # tuning knob (see DESIGN.md section 5)
        self.arena = FlatArena(model.parameters(), process_group, world_size, bucket_mb=bucket_mb)
        self.overlap = overlap   # bucketed all-reduce on a side stream during the backward pass (False: one call after it)
        if self.arena.flat_p.device.type != "cuda":
            raise RuntimeError("TrainStep needs the model on a CUDA (sm_90a) device; there is no CPU fallback")
        self.world = self.arena.world
        self.steps = 0
        self.label_smoothing = float(label_smoothing)
        self.accum_steps = int(accum_steps)
        if self.accum_steps < 1:
            raise ValueError("accum_steps must be >= 1")
        self._micro = 0   # micro-batches accumulated since the last update
        self._acc = torch.zeros_like(self.arena.flat_g) if self.accum_steps > 1 else None
        self.clip_grad = clip_grad
        self._clip = None
        if clip_grad is not None:
            dev = self.arena.flat_p.device
            self._clip = torch.ones(2, dtype=torch.float32, device=dev)   # {coefficient, total norm}
            self._clip_scratch = torch.empty(ops_clip_blocks(), dtype=torch.float32, device=dev)
        if optimizer == "adamw":
            arena = self.arena
            rule = no_decay or model_no_decay_rule(model)
            names = {p.data_ptr(): n for n, p in model.named_parameters()}
            arena.flat_wd = torch.zeros_like(arena.flat_p)
            for p, o in zip(arena.params, arena.offsets):
                if not rule(names.get(p.data_ptr(), ""), p):
                    arena.flat_wd[o:o + p.numel()] = weight_decay
        if optimizer in ("adamw", "adam"):
            arena = self.arena
            arena.flat_v = torch.zeros_like(arena.flat_p)
            self._hyper = torch.tensor([lr, 0.0, 0.0, 1.0, 1.0], dtype=torch.float32, device=arena.flat_p.device)
        if broadcast:
            self.arena.broadcast(model.buffers())
        weight_cache.bump()

    # ------------------------------------------------------------------------------------------------ eager step
    def _fwd_bwd(self, images, labels, last=True):
        """Forward, loss, backward AND the gradient all-reduce (overlapped with the backward pass when ``overlap``).
        With gradient accumulation only the ``last`` micro-batch of a group reduces (the sum of the group's gradients)."""
        model, arena = self.model, self.arena
        logits, tape = self.engine.forward(model, images, True, True)
        loss, dlogits, correct = ops.softmax_xent(logits, labels, want_grad=True, ld_d=padded_classes(logits.shape[1]),
                                                  label_smoothing=self.label_smoothing, loss_scale=1.0 / self.accum_steps)
        if self.accum_steps > 1:
            self.engine.backward(model, tape, dlogits, sink=arena.grad_view)
            if last:
                arena.flat_g.add_(self._acc)
                self._acc.zero_()
                arena.all_reduce_grads()
            else:
                self._acc.add_(arena.flat_g)
            return loss, correct
        if self.world > 1 and self.overlap:
            arena.begin_backward()
            self.engine.backward(model, tape, dlogits, sink=_GradSink(arena))
            arena.finish_backward()
        else:
            self.engine.backward(model, tape, dlogits, sink=arena.grad_view)
            arena.all_reduce_grads()
        return loss, correct

    @property
    def grad_norm(self):
        """Total gradient norm of the last step (device scalar), when clip_grad is set."""
        return None if self._clip is None else self._clip[1]

    def _update(self, lr, lr_dev=None):
        arena = self.arena
        if self._clip is not None:
            ops.grad_clip_coef(arena.flat_g, self.clip_grad, gscale=arena.grad_scale, out=self._clip, scratch=self._clip_scratch)
        if self.optimizer == "adamw":
            if lr != self._hyper_lr():
                self._hyper[0:1].fill_(float(lr))
                self._hyper_lr_value = float(lr)
            ops.adamw_(arena.flat_p, arena.flat_g, arena.flat_m, arena.flat_v, arena.flat_wd, self._hyper, self.betas[0],
                       self.betas[1], self.eps, gscale=arena.grad_scale, clip=self._clip)
            weight_cache.bump()
            return
        if self.optimizer == "adam":
            if lr != self._hyper_lr():
                self._hyper[0:1].fill_(float(lr))
                self._hyper_lr_value = float(lr)
            ops.adam_(arena.flat_p, arena.flat_g, arena.flat_m, arena.flat_v, self._hyper, self.betas[0], self.betas[1],
                      self.eps, self.weight_decay, gscale=arena.grad_scale, clip=self._clip)
            weight_cache.bump()
            return
        # momentum buffer starts at zero, so "buf = mu*buf + g" already equals torch's first-step "buf = g"
        ops.sgd_momentum_(arena.flat_p, arena.flat_g, arena.flat_m, lr, self.momentum, self.weight_decay,
                          gscale=arena.grad_scale, first_step=False, lr_dev=lr_dev, clip=self._clip)
        weight_cache.bump()  # parameters changed behind autograd's back -> repack bf16 operands on next use

    def _hyper_lr(self):
        return getattr(self, "_hyper_lr_value", self.lr)

    def step_eager(self, images, labels, lr=None):
        if not self.model.training:
            self.model.train()
        last = self._micro + 1 == self.accum_steps
        loss, correct = self._fwd_bwd(images, labels, last)
        self._micro = 0 if last else self._micro + 1
        if last:
            self._update(self.lr if lr is None else lr)
            self.steps += 1
        return loss, correct

    # ------------------------------------------------------------------------------------------------ CUDA-graph step
    def capture(self, images, labels):
        """Capture fwd + loss + bwd + gradient all-reduce + update into ONE CUDA graph with static input buffers of the given
        shapes (world > 1: the NCCL collectives of the gradient buckets are graph nodes on a side stream)."""
        if not self.model.training:
            self.model.train()
        dev = self.arena.flat_p.device
        # (a decoded uint8 NHWC batch stays uint8: ToTensor + Normalize run inside the step, see ops.stem_s2d_u8)
        self._g_images = torch.empty_like(images, dtype=torch.uint8 if images.dtype == torch.uint8 else torch.float32, device=dev)
        self._g_labels = torch.empty_like(labels, device=dev)
        self._g_images.copy_(images)
        self._g_labels.copy_(labels)
        self._lr_dev = torch.full((1,), float(self.lr), dtype=torch.float32, device=dev)
        # The warm-up below runs two real steps (first-launch attribute calls, allocator growth).  They must not perturb
        # the caller's model: parameters, optimizer state, AdamW step counters and every buffer (BatchNorm running
        # statistics, num_batches_tracked) are snapshotted and restored, so capture() with a dummy batch is side-effect free.
        arena = self.arena
        saved = [t.clone() for t in (arena.flat_p, arena.flat_m)]
        saved_v = arena.flat_v.clone() if hasattr(arena, "flat_v") else None
        saved_hyper = self._hyper.clone() if hasattr(self, "_hyper") else None
        saved_bufs = [b.clone() for b in self.model.buffers()]
        saved_steps = self.steps
        if self._micro != 0:
            raise RuntimeError("capture() in the middle of a gradient-accumulation group")
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                for m in range(self.accum_steps):
                    self._fwd_bwd(self._g_images, self._g_labels, m + 1 == self.accum_steps)
                self._update(self.lr, self._lr_dev)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        with torch.no_grad():
            arena.flat_p.copy_(saved[0])
            arena.flat_m.copy_(saved[1])
            if saved_v is not None:
                arena.flat_v.copy_(saved_v)
            if saved_hyper is not None:
                self._hyper.copy_(saved_hyper)
            for b, sb in zip(self.model.buffers(), saved_bufs):
                b.copy_(sb)
        self.steps = saved_steps
        weight_cache.bump()
        # ONE graph for the whole step; with world > 1 it contains the NCCL all-reduces of the gradient buckets on their side
        # stream ("thread_local": the NCCL watchdog thread's CUDA calls must not invalidate the capture)
        self._graph_fb = torch.cuda.CUDAGraph()
        self._graph_up = None
        self._graph_acc = None
        if self.accum_steps > 1:
            # the micro-batches before the last of a group: forward + backward + accumulate, no collective, no update
            self._graph_acc = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._graph_acc, capture_error_mode="thread_local"):
                self._g_loss_acc, self._g_correct_acc = self._fwd_bwd(self._g_images, self._g_labels, False)
            self._acc.zero_()
        with torch.cuda.graph(self._graph_fb, capture_error_mode="thread_local"):
            self._g_loss, self._g_correct = self._fwd_bwd(self._g_images, self._g_labels, True)
            self._update(self.lr, self._lr_dev)
        self._captured_shape = (tuple(images.shape), tuple(labels.shape))
        return self

    def step(self, images, labels, lr=None):
        """One training step on this rank's shard. Returns (loss [1] fp32 device tensor, correct int32 [B]).
        Replays the captured graphs when ``capture()`` was called with matching shapes, else runs eagerly."""
        if getattr(self, "_graph_fb", None) is None or (tuple(images.shape), tuple(labels.shape)) != self._captured_shape:
            return self.step_eager(images, labels, lr)
        if images.data_ptr() != self._g_images.data_ptr():
            self._g_images.copy_(images, non_blocking=True)
        if labels.data_ptr() != self._g_labels.data_ptr():
            self._g_labels.copy_(labels, non_blocking=True)
        if lr is not None and lr != self.lr:
            self.lr = lr
            self._lr_dev.fill_(float(lr))
            if self.optimizer in ("adamw", "adam"):
                self._hyper[0:1].fill_(float(lr))
                self._hyper_lr_value = float(lr)
        if self._micro + 1 < self.accum_steps:
            self._micro += 1
            self._graph_acc.replay()
            return self._g_loss_acc, self._g_correct_acc
        self._micro = 0
        self._graph_fb.replay()
        self.steps += 1
        # the replay updated the parameters behind autograd's back (and repacked the bf16 operands from the PRE-update
        # values at its start): any forward outside the graph must repack first
        weight_cache.bump()
        return self._g_loss, self._g_correct

    # ------------------------------------------------------------------------------------------- checkpoint / resume
    def optimizer_state_dict(self):
        """The fused optimizer's state in ``torch.optim`` format: what ``optimizer.state_dict()`` of the reference's
        ``torch.optim.SGD(model.parameters(), ...)`` (resnet/train.py:96) or grouped ``AdamW`` (convNext/train.py:102,
        swin utils/optimizer.py) would hold after the same steps - parameters indexed in ``model.parameters()`` order - so it
        drops into the reference's checkpoint dict (swin_transformer/utils/torch_utils.py ``save_checkpoint``:
        {'model', 'optimizer', 'lr_scheduler', 'max_accuracy', 'scaler', 'epoch', 'config'}) and into a real torch optimizer."""
        arena = self.arena
        state = {}
        decay, nodecay = [], []
        for i, (prm, o) in enumerate(zip(arena.params, arena.offsets)):
            n = prm.numel()
            if self.optimizer == "sgd":
                if self.steps > 0:
                    state[i] = {"momentum_buffer": arena.flat_m[o:o + n].view_as(prm).clone()}
            else:
                if self.steps > 0:
                    state[i] = {"step": torch.tensor(float(self.steps)), "exp_avg": arena.flat_m[o:o + n].view_as(prm).clone(),
                                "exp_avg_sq": arena.flat_v[o:o + n].view_as(prm).clone()}
                if self.optimizer == "adamw":
                    (decay if float(arena.flat_wd[o]) != 0.0 else nodecay).append(i)
        if self.optimizer == "sgd":
            groups = [{"lr": self.lr, "momentum": self.momentum, "dampening": 0, "weight_decay": self.weight_decay,
                       "nesterov": False, "params": list(range(len(arena.params)))}]
        elif self.optimizer == "adam":
            groups = [{"lr": self._hyper_lr(), "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.weight_decay,
                       "amsgrad": False, "params": list(range(len(arena.params)))}]
        else:
            base = {"lr": self._hyper_lr(), "betas": tuple(self.betas), "eps": self.eps, "amsgrad": False}
            groups = [dict(base, weight_decay=self.weight_decay, params=decay), dict(base, weight_decay=0.0, params=nodecay)]
        return {"state": state, "param_groups": groups}

    def load_optimizer_state_dict(self, sd):
        """Inverse of ``optimizer_state_dict`` (also accepts the state dict of a torch optimizer built over
        ``model.parameters()`` in order): resume of the reference's ``load_checkpoint``."""
        arena = self.arena
        steps = 0
        with torch.no_grad():
            arena.flat_m.zero_()
            if hasattr(arena, "flat_v"):
                arena.flat_v.zero_()
            for i, st in sd["state"].items():
                o, prm = arena.offsets[int(i)], arena.params[int(i)]
                n = prm.numel()
                if self.optimizer == "sgd":
                    if st.get("momentum_buffer") is not None:
                        arena.flat_m[o:o + n].copy_(st["momentum_buffer"].reshape(-1))
                        steps = max(steps, 1)
                else:
                    arena.flat_m[o:o + n].copy_(st["exp_avg"].reshape(-1))
                    arena.flat_v[o:o + n].copy_(st["exp_avg_sq"].reshape(-1))
                    steps = max(steps, int(float(st["step"])))
        lr = sd["param_groups"][0]["lr"]
        self.lr = float(lr)
        if self.optimizer in ("adamw", "adam"):
            b1, b2 = self.betas
            self._hyper.copy_(torch.tensor([self.lr, 1.0 - b1 ** steps, 1.0 - b2 ** steps, b1 ** steps, b2 ** steps],
                                           dtype=torch.float32))
            self._hyper_lr_value = self.lr
            self.steps = steps
        elif steps and self.steps == 0:
            self.steps = steps   # (SGD keeps no step counter; only "has stepped" matters)
        if getattr(self, "_lr_dev", None) is not None:
            self._lr_dev.fill_(self.lr)

    @property
    def static_inputs(self):
        """(images, labels) buffers the captured graph reads; fill them directly to avoid the device-to-device copy."""
        return self._g_images, self._g_labels
