"""Whole-step CUDA-graph capture of the relight training step.

Eagerly, one step is ~1000 kernel launches (compacted-list bookkeeping, MLP heads, shading epilogue, autograd,
Adam) and is bound by host launch latency, not by the GPU.  Here every dynamically-sized list of the primary march is
given a static capacity (rows past the real total are zero padding; overflow is counted on the device and checked by
the host), host-drawn random numbers are written into static device buffers before each replay, and the whole
forward + loss + backward + (optional gradient all-reduce) + Adam is captured once into a CUDA graph and replayed.

Anything the host changes from step to step must live in device memory to reach a replay: ray batch / light indices
(copied in by ``run``), the host-drawn randoms (staged by ``run``), learning rates (``lr_tensors`` + ``scale_lr``), and
any loss weight that ``loss_fn`` varies over the iterations (the reference decays its TV weights,
train_tensoIR.py:277-282) — keep those in 0-dim device tensors and update them in place between replays; Python floats
are baked in at capture.  Grid maintenance (updateAlphaMask / shrink / upsample) needs a new capture (``run`` checks).

Capacities can never silently change the computation: every list records its real length on the device, a step whose
lists did not fit raises a device-side flag that (i) turns the optimizer update of that very step into an exact no-op
(``found_inf`` of the fused Adam: parameters, moments and step counters untouched) and (ii) is read back by the host a
step later, which then re-captures the graph with larger lists and REDOES the same batch.  The host also watches the
high-water marks and grows the lists before they fill up (``grow_at``), so an overflow needs a >20 % jump from one batch to
the next.  ``redone`` / ``recaptures`` count what happened; bench.py fails if a timed step had to be redone.

Numerics are those of the eager path except for (i) the device-side xyz-noise draw, which has the padded shape and
therefore a different random stream, and (ii) atomics ordering.  Parity tests run the eager path.
"""
from __future__ import annotations

import torch

from . import _lib
from .device_field import mark_parameters_updated
from .renderer import Renderer_TensoIR_train


def lr_tensors(param_groups, device):
    """Optimizer param groups with their learning rates turned into 0-dim fp32 tensors on ``device`` (what
    ``torch.optim.Adam(..., capturable=True)`` reads on the device at every replay), so that learning-rate decay keeps
    working under CUDA-graph replay (:meth:`StaticTrainStep.scale_lr`)."""
    out = []
    for grp in param_groups:
        grp = dict(grp)
        grp["lr"] = torch.as_tensor(float(grp["lr"]), dtype=torch.float32, device=device)
        out.append(grp)
    return out


class StaticTrainStep:
    LISTS = ("cap_valid", "cap_app")      # surface hits are not a list any more (relight_utils.render_hits)

    def __init__(self, model, optimizer, n_rays, n_samples, args, loss_fn, *, sample_method="stratified_sampling",
                 cap_valid=None, cap_app=None, grad_bucket=None, device=None, grow_at=0.8, headroom=1.5, lag=2):
        self.model, self.opt, self.args, self.loss_fn = model, optimizer, args, loss_fn
        self.n_rays, self.n_samples, self.sample_method = int(n_rays), int(n_samples), sample_method
        self.bucket = grad_bucket
        dev = device or model.device
        self.dev = dev
        self.grow_at, self.headroom, self.lag = float(grow_at), float(headroom), max(1, int(lag))
        self.rays = torch.zeros(n_rays, 6, device=dev)
        self.light_idx = torch.zeros(n_rays, 1, dtype=torch.int32, device=dev)
        n_dirs = model.envmap_h * model.envmap_w
        self.static = {"cap_valid": int(cap_valid or 256 * n_rays), "cap_app": int(cap_app or 16 * n_rays),
                       "sec_per_slot": 4,
                       "jitter": torch.zeros(n_rays, 1, device=dev),
                       "dirs": torch.zeros(n_dirs, 3, device=dev),
                       # real list lengths of the last step: valid samples, appearance samples, (unused), secondary
                       # appearance samples (device side; the host reads them `lag` steps late)
                       "stats": torch.zeros(4, dtype=torch.int64, device=dev),
                       "overflow_step": torch.zeros((), dtype=torch.int64, device=dev),
                       "overflow": torch.zeros((), dtype=torch.int64, device=dev)}
        # found_inf of torch's fused / capturable Adam: 1.0 -> the whole update (parameters, moments, step counters)
        # is skipped.  Raised by a list overflow, so an overflowed step leaves the model exactly as it was.
        self.found_inf = torch.zeros((), dtype=torch.float32, device=dev)
        # 1.0 while capture() warms up: those eager executions must not train on whatever the input buffers hold
        self.force_skip = torch.zeros((), dtype=torch.float32, device=dev)
        self.graph = None
        self.loss = None
        self.launches_per_replay = 0
        self.redone = 0            # steps that overflowed (no-op on the device) and were executed again
        self.recaptures = 0        # graph re-captures with larger lists (overflow or high-water mark)
        self._step = 0
        ring = self.lag + 1
        # ring of pinned staging slots: the host never rewrites a slot whose copies may still be in flight
        self._slots = [{"jitter": torch.zeros(n_rays, 1).pin_memory(), "dirs": torch.zeros(n_dirs, 3).pin_memory(),
                        "stats": torch.zeros(5, dtype=torch.int64).pin_memory(), "event": None, "batch": None}
                       for _ in range(ring)]

    # ------------------------------------------------------------------------------------------------ capacities
    @torch.no_grad()
    def calibrate(self, batches, headroom=None):
        """Size the static lists from eager marches over a few representative batches (max count x headroom).
        The lists grow by themselves later (``run``), so this only has to be a sensible start."""
        from . import primary
        headroom = float(headroom or self.headroom)
        self.model.__dict__.pop("_tir_static", None)
        nv = na = 0
        for rays, _ in batches:
            m = primary.march(self.model, rays.to(self.dev).float(), True, self.n_samples)
            nv = max(nv, int(m["xn"].shape[0]))
            na = max(na, int((m["weight"] > self.model.rayMarch_weight_thres).sum().item()))
        self._set_caps(int(headroom * nv) + 4096, int(headroom * na) + 1024)
        return self.capacities()

    def _set_caps(self, cap_valid, cap_app, *_unused):
        self.static["cap_valid"] = int(min(cap_valid, self.n_rays * max(self.n_samples, 1)))
        self.static["cap_app"] = int(min(cap_app, self.static["cap_valid"]))

    def capacities(self):
        return tuple(self.static[k] for k in self.LISTS)

    # -- host side of one step: the reference's CPU draws, in the reference's order, into the static buffers
    def _stage_host_randoms(self, slot):
        slot["jitter"].copy_(torch.rand(self.n_rays, 1))                                    # tensorBase:714-718
        slot["dirs"].copy_(self.model.gen_light_incident_dirs(method=self.sample_method))   # tensorBase:511-526
        self.static["jitter"].copy_(slot["jitter"], non_blocking=True)
        self.static["dirs"].copy_(slot["dirs"], non_blocking=True)

    def _body(self):
        st = self.static
        st["overflow_step"].zero_()
        ret = Renderer_TensoIR_train(self.rays, None, self.light_idx, self.model, N_samples=self.n_samples,
                                     white_bg=True, is_train=True, is_relight=True, sample_method=self.sample_method,
                                     chunk_size=160000, device=self.dev, args=self.args)
        loss = self.loss_fn(ret, self.model)
        self.ret = ret                    # the captured forward's outputs: after a replay they hold that step's values
        loss.backward()
        flag = torch.maximum((st["overflow_step"] > 0).to(torch.float32), self.force_skip)
        if self.bucket is not None:
            # the flag rides in the bucket's spare slot: one rank's overflow makes every rank skip the same step
            self.bucket.extra[0].copy_(flag)
            self.bucket.all_reduce_mean()
            flag = (self.bucket.extra[0] > 0).to(torch.float32)
        self.found_inf.copy_(flag)
        st["overflow"].add_((st["overflow_step"] > 0).to(torch.int64))
        self.opt.step()
        return loss

    def capture(self, warmup=3, capture_error_mode="global"):
        """Warm up eagerly on a side stream (allocations, cudaFuncSetAttribute, cuBLAS handles), then capture."""
        self.model.__dict__["_tir_static"] = self.static
        self.opt.found_inf = self.found_inf           # read by Adam.step() (fused / capturable implementations)
        _lib.load()
        # warm-up and capture run on the SAME side stream: autograd's AccumulateGrad nodes remember the stream they
        # were created on, and a mismatch with the capturing stream would need a cross-stream sync that is illegal
        # during capture
        s = getattr(self, "_stream", None) or torch.cuda.Stream()
        self._stream = s
        self.force_skip.fill_(1.0)
        s.wait_stream(torch.cuda.current_stream())
        # FusedAdam(clear_grad=True) keeps every gradient zeroed IN PLACE: the buffers created by the first warm-up step
        # are the ones the captured kernels accumulate into (no per-step allocation / memset / AccumulateGrad pass)
        keep_grads = bool(getattr(self.opt, "clear_grad", False))
        with torch.cuda.stream(s):
            for _ in range(max(warmup, 1)):
                self._stage_host_randoms(self._slots[0])
                self.opt.zero_grad(set_to_none=not keep_grads)
                self._body()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self._stage_host_randoms(self._slots[0])
        self.graph = torch.cuda.CUDAGraph()
        self.opt.zero_grad(set_to_none=not keep_grads)
        l0 = _lib.launch_count
        with torch.cuda.graph(self.graph, stream=s, capture_error_mode=capture_error_mode):
            self.loss = self._body()
        self.launches_per_replay = _lib.launch_count - l0
        self.force_skip.zero_()
        self.static["overflow"].zero_()
        torch.cuda.synchronize()
        for slot in self._slots:
            slot["event"], slot["batch"] = None, None
        # The captured kernels hold raw pointers into buffers owned elsewhere (the sample-list scratch, the alpha-mask
        # and VM shadows).  Keep references so that a later eager call that re-sizes / rebuilds them cannot hand the
        # memory back to the allocator while this graph can still be replayed.
        df = self.model.__dict__.get("_tir_device_field")
        self._keepalive = [self.model.__dict__.get("_tir_scratch"), self.model.alphaMask,
                           None if df is None else (df.dplane, df.dline, df.aplane, df.aline, df.amask, df.acell)]
        self._captured_for = self._model_signature()
        return self

    def _model_signature(self):
        """Identity of everything the graph baked in by address: grid maintenance (updateAlphaMask / shrink /
        upsample_volume_grid, train_tensoIR.py:386-422) replaces these objects and requires a new capture."""
        m = self.model
        vm = list(m.density_plane) + list(m.density_line) + list(m.app_plane) + list(m.app_line)
        return (id(m.alphaMask), tuple((p.data_ptr(), tuple(p.shape)) for p in vm))

    # ------------------------------------------------------------------------------------------------ replay
    def _launch(self, rays, light_idx, slot):
        self.rays.copy_(rays, non_blocking=True)
        self.light_idx.copy_(light_idx.reshape(-1, 1), non_blocking=True)
        self._stage_host_randoms(slot)
        self.graph.replay()
        slot["stats"][:4].copy_(self.static["stats"], non_blocking=True)
        slot["stats"][4:5].copy_(self.static["overflow_step"].reshape(1), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        slot["event"], slot["batch"] = ev, (rays, light_idx)
        mark_parameters_updated()        # the replayed optimizer step is invisible to the host-side bookkeeping
        _lib.launch_count += self.launches_per_replay

    def _inspect(self, slot):
        """Look at a finished step: -> (overflowed, grow) with grow = new capacities or None."""
        slot["event"].synchronize()
        n_valid, n_app, _, n_sec, over = (int(v) for v in slot["stats"].tolist())
        slot["event"] = None
        caps = self.capacities()
        seen = (n_valid, n_app)
        old = getattr(self, "_seen", (0, 0, 0))
        self._seen = tuple(max(a, b) for a, b in zip(old, (n_valid, n_app, n_sec)))
        want = list(caps)
        for i in range(2):
            if seen[i] > self.grow_at * caps[i]:
                want[i] = int(self.headroom * seen[i]) + 64
        slots = self.n_rays * self.static["dirs"].shape[0]
        sec_cap = max(1 << 16, self.static["sec_per_slot"] * slots)
        if n_sec > self.grow_at * sec_cap:          # secondary appearance scratch: rows per (ray, direction) slot
            self.static["sec_per_slot"] = int(self.headroom * n_sec / max(1, slots)) + 1
            return bool(over), tuple(want)
        return bool(over), (None if tuple(want) == caps else tuple(want))

    def _recapture(self, caps):
        import sys
        sys.stderr.write(f"StaticTrainStep: re-capture, lists {self.capacities()} -> {tuple(caps)}, secondary rows per "
                         f"slot {self.static['sec_per_slot']}, longest seen {getattr(self, '_seen', None)}\n")
        self.graph = None
        before = (self.capacities(), self.static["sec_per_slot"])
        self._set_caps(*caps)
        if getattr(self, "_last_grow", None) == (before, (self.capacities(), self.static["sec_per_slot"])):
            raise RuntimeError(f"static lists {before} overflow and cannot grow any further")
        self._last_grow = (before, (self.capacities(), self.static["sec_per_slot"]))
        self.recaptures += 1
        self.capture(warmup=1)

    def _settle(self, slot):
        """Host-side follow-up of one finished step (read ``lag`` steps late): grow the lists when a high-water mark
        came close to its capacity; an overflowed step (a no-op on the device) is redone after the re-capture."""
        if slot["event"] is None:
            return
        batch = slot["batch"]
        over, grow = self._inspect(slot)
        if over and grow is None:
            grow = tuple(int(self.headroom * c) + 64 for c in self.capacities())
        if grow is not None:
            torch.cuda.synchronize()
            pending = [s for s in self._slots if s["event"] is not None]
            redo = [batch] if over else []
            for s in pending:                        # steps launched after the inspected one, already finished
                o, _ = self._inspect(s)
                if o:
                    redo.append(s["batch"])
            self._recapture(grow)
            for rays, li in redo:
                self.redone += 1
                self._launch(rays, li, self._slots[0])
                self._settle_now(self._slots[0])

    def _settle_now(self, slot):
        torch.cuda.synchronize()
        self._settle(slot)

    def run(self, rays, light_idx):
        """One training step.  ``rays`` / ``light_idx`` may live on the host (pinned) or on the device."""
        if self.graph is None:
            raise RuntimeError("StaticTrainStep.run() before capture()")
        if self._model_signature() != self._captured_for:
            raise RuntimeError("the model's alpha mask or VM factors were replaced (updateAlphaMask / shrink / "
                               "upsample_volume_grid) after capture(): build and capture a new StaticTrainStep")
        slot = self._slots[self._step % len(self._slots)]
        self._settle(slot)                          # the step that used this slot `lag + 1` calls ago
        self._step += 1
        self._launch(rays, light_idx, slot)
        return self.loss

    def reserve(self, factor=2.0):
        """Make every list at least ``factor`` x the largest length seen so far (re-captures if something grows).
        Call it after a few warm-up steps, outside any region whose timing matters."""
        self.flush()
        seen = getattr(self, "_seen", None)
        if seen is None:
            return self.capacities()
        caps = self.capacities()
        want = tuple(max(c, int(factor * v) + 64) for c, v in zip(caps, seen[:2]))
        self._set_caps(*want)
        if self.capacities() != caps:
            new = self.capacities()
            self._set_caps(*caps)
            self._recapture(new)
        return self.capacities()

    def flush(self):
        """Settle every step still in flight (end of training / before reading results that must be exact)."""
        for _ in range(len(self._slots)):
            for slot in self._slots:
                if slot["event"] is not None:
                    self._settle_now(slot)

    def scale_lr(self, factor: float):
        """The train loop's per-iteration decay ``param_group['lr'] = param_group['lr'] * lr_factor``
        (train_tensoIR.py:380-381) for a captured step: a Python-float learning rate is baked into the graph at capture,
        so the rates must be 0-dim device tensors (see :func:`lr_tensors`) and are scaled IN PLACE here, between
        replays, where the next replay reads them."""
        for grp in self.opt.param_groups:
            lr = grp["lr"]
            if not isinstance(lr, torch.Tensor):
                raise TypeError("scale_lr() needs tensor learning rates: build the optimizer from "
                                "static_step.lr_tensors(model.get_optparam_groups(...), device)")
            lr.mul_(factor)

    def overflowed(self) -> int:
        """Number of replays whose lists exceeded the static capacities (each was a no-op and has been, or will be,
        redone by ``run`` / ``flush``).  Host sync."""
        return int(self.static["overflow"].item())

    def release(self):
        self.model.__dict__.pop("_tir_static", None)
        if getattr(self.opt, "found_inf", None) is self.found_inf:
            del self.opt.found_inf
