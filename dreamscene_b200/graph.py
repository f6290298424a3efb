"""A training step replayed from two CUDA graphs (DESIGN.md section 0, f8).

DreamScene's step is render -> guidance loss (SDS, not capturable) -> backward -> optimizer steps.  With the native
kernels the step's device work is short enough that the host's launch cost bounds it; ``StepGraph`` captures the
native parts as two graphs and runs the user's loss eagerly between them:

    sg = StepGraph(groups, optimizers, views=B, height=H, width=W)
    out = sg.render(settings_list, shs_aug=..., scale_aug=..., seed=...)   # graph 1: B views + the disparity
    loss = user_loss(out.image, out.disp, out.scales)                     # eager
    loss.backward()
    sg.step()       # graph 2: render backward, disparity backward, every GaussianAdam step
    sg.check()      # raises PairCapacityOverflow if a replay since the last check overflowed its key buffer

The per-step values a replay must not freeze - cameras, bg, tanfov, sh_degree, the augmentation flags, the seed, the
disparity focal lengths and the Adam scalars - live in static device buffers that ``render()`` / ``step()`` rewrite
before each replay (include/b200gsr_step.h).  A step equals render_scene + disparity_from_depth_alpha + backward +
GaussianAdam.step() for the same values; in deterministic mode bit for bit.

The first ``render()`` of a layout runs one eager forward and backward (which measure the pair capacity and set up
the library) and then captures.  The layout - P, the group tensors, the optimizer state tensors, the per-view
scale_modifier and deterministic mode - is compared on the host at every ``render()``; a change (densify / prune)
re-captures.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import NamedTuple, Sequence

import torch

from . import _lib
from . import optim as O
from . import rasterizer as R
from . import scene as S

_SEED_WORDS = 8             # the uint64 seed, padded so the view records start 32-byte aligned
_VIEW_WORDS = 8             # sizeof(b200gsr_step_view) / 4


class StepOutputs(NamedTuple):
    """Static tensors, overwritten by the next render().  image / disp / alpha / scales are leaves that require grad:
    the loss's gradients reach step() through their .grad."""
    image: torch.Tensor     # [B,3,H,W]
    disp: torch.Tensor      # [B,1,H,W]
    alpha: torch.Tensor     # [B,1,H,W]
    radii: torch.Tensor     # [B,P] int32
    scales: torch.Tensor    # [B,P,3] the augmented scales (for the scale loss)


class StepGraph:
    """One training step of `views` views of height x width over the parameter groups `groups` (as render_scene),
    with the GaussianAdam optimizers `optimizers` over their leaves, replayed from CUDA graphs."""

    def __init__(self, groups: Sequence, optimizers: Sequence, *, views: int, height: int, width: int):
        self.groups = list(groups)
        self.optimizers = list(optimizers)
        self.B, self.H, self.W = int(views), int(height), int(width)
        if not 1 <= self.B <= _lib.MAX_VIEWS:
            raise ValueError(f"StepGraph: views must be in 1..{_lib.MAX_VIEWS}")
        for opt in self.optimizers:
            if not isinstance(opt, O.GaussianAdam):
                raise TypeError(f"StepGraph: only GaussianAdam optimizers can be replayed, got {type(opt).__name__}")
        self._key = None
        self._report = None         # device [2]: max pair count, overflowed replays; kept across re-captures
        self._scratch_key = None
        self.d_means2D = None       # [B,P,3] per-view screen-space gradients of the last step (densification stats)
        self.grads = None           # per group {leaf name: its gradient of the last step} (the update graph's buffers)

    # ---- per-step values -----------------------------------------------------------------------------------------
    def _views(self, settings, shs_aug, scale_aug, M):
        B, H, W = S._check_settings(settings)
        if (B, H, W) != (self.B, self.H, self.W):
            raise ValueError(f"StepGraph: built for {self.B} views of {self.H}x{self.W}, got {B} of {H}x{W}")
        shs = S._view_flags(shs_aug, B, "shs_aug")
        sca = S._view_flags(scale_aug, B, "scale_aug")
        rec = []
        for v, s in enumerate(settings):
            deg, tx, ty = int(s.sh_degree), float(s.tanfovx), float(s.tanfovy)
            if not (0 <= deg <= 3 and (deg + 1) ** 2 <= M):
                raise ValueError(f"StepGraph: view {v}: sh_degree {deg} needs (deg+1)^2 <= M = {M}")
            if not (tx > 0 and ty > 0 and tx < float("inf") and ty < float("inf")):
                raise ValueError(f"StepGraph: view {v}: tanfovx / tanfovy must be positive and finite")
            rec.append((tx, ty, S.NOISE_COEF if shs[v] else 0.0, S.NOISE_COEF if sca[v] else 0.0, deg))
        return rec

    def _layout(self, flat, P, M, settings, det):
        ptrs = tuple((t.data_ptr(), tuple(t.shape)) for t in flat)
        states = []
        for opt in self.optimizers:
            for group in opt.param_groups:
                for p in group["params"]:
                    st = opt.state.get(p, {})
                    states.append((id(p), st["exp_avg"].data_ptr() if st else 0, st["exp_avg_sq"].data_ptr() if st else 0))
        return (P, M, ptrs, tuple(states), tuple(float(s.scale_modifier) for s in settings), det)

    def _upload(self, settings, rec, seed, focal):
        """One pinned staging tensor, one non_blocking copy of it (plus one device concatenation when the cameras
        are CUDA tensors).  The caching host allocator keeps the staging buffer alive until its copy has run."""
        B, dev = self.B, self._dev.device
        stage = torch.empty(self._dev.numel(), dtype=torch.float32, pin_memory=True)
        stage[:2].view(torch.int64)[0] = int(seed)
        views = stage[_SEED_WORDS:_SEED_WORDS + _VIEW_WORDS * B].view(B, _VIEW_WORDS)
        views[:, :4] = torch.tensor([r[:4] for r in rec], dtype=torch.float64)
        views[:, 4:].view(torch.int32)[:, 0] = torch.tensor([r[4] for r in rec], dtype=torch.int32)
        f0 = _SEED_WORDS + _VIEW_WORDS * B
        stage[f0:f0 + B] = torch.tensor([float(f) for f in focal], dtype=torch.float64)
        cams = ([s.viewmatrix for s in settings] + [s.projmatrix for s in settings] + [s.campos for s in settings] +
                [s.bg for s in settings])
        c0 = self._cam0
        if all(c.device.type == "cpu" for c in cams):
            torch.cat([c.detach().reshape(-1).float() for c in cams], out=stage[c0:])
            self._dev.copy_(stage, non_blocking=True)
        else:
            self._dev[:c0].copy_(stage[:c0], non_blocking=True)
            torch.cat([c.detach().reshape(-1).to(dev, torch.float32) for c in cams], out=self._dev[c0:])

    def _adam_records(self):
        """-> [(p, grad buffer, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, step tensor)] of every optimizer
        parameter, with torch's state created as GaussianAdam.step() creates it."""
        out = []
        for opt in self.optimizers:
            for group in opt.param_groups:
                O._check_group(group)
                lr, (b1, b2), eps = group["lr"], group["betas"], group["eps"]
                for p in group["params"]:
                    g = self._grad_of.get(id(p))
                    if g is None:
                        raise ValueError("StepGraph: every optimizer parameter must be a raw leaf of the groups")
                    if not p.requires_grad:
                        raise ValueError("StepGraph: an optimizer parameter does not require grad: GaussianAdam.step() "
                                         "would skip it, the update graph would step it")
                    state = opt.state[p]
                    if len(state) == 0:
                        state["step"] = torch.tensor(0.0, dtype=torch.float32)
                        state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                        state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    m, v, st = state["exp_avg"], state["exp_avg_sq"], state["step"]
                    if not (p.dtype == m.dtype == v.dtype == st.dtype == torch.float32 and p.is_contiguous()
                            and m.is_contiguous() and v.is_contiguous() and st.is_cpu and p.shape == m.shape == v.shape
                            and p.device == m.device == v.device == self._dev.device):
                        O._refuse(p, g, m, v, st, self._dev.device)
                    out.append((p, g, m, v, lr, b1, b2, eps, st))
        return out

    # ---- capture -------------------------------------------------------------------------------------------------
    def _capture(self, flat, P, M, settings, det, values):
        """Allocate the static buffers, upload this step's `values` = (records, seed, focal), run the step's render
        and backward eagerly once (measuring the pair capacity), then capture both graphs."""
        B, H, W = self.B, self.H, self.W
        dev = flat[0].device
        lib, ptr = _lib.load(), _lib.ptr
        self._graphs = None
        ng = len(self.groups)
        raw = [[_lib.prepare(t.detach()) for t in flat[6 * k:6 * k + 6]] for k in range(ng)]
        if any(r.data_ptr() != t.data_ptr() for r, t in zip([t for ts in raw for t in ts], flat)):
            raise ValueError("StepGraph: the group tensors must be float32, contiguous and 16-byte aligned "
                             "(a copy would freeze their values into the graph)")
        Hs = _lib.stacked_height(B, H, W)
        Hp = Hs // B
        self._cam0 = c0 = (_SEED_WORDS + _VIEW_WORDS * B + B + 63) // 64 * 64
        # [seed | B view records | B focal lengths | pad | B viewmatrix, B projmatrix, B campos, B bg]
        self._dev = torch.zeros(c0 + B * 38, dtype=torch.float32, device=dev)
        seed_t = self._dev[:2].view(torch.int64)
        views_t = self._dev[_SEED_WORDS:_SEED_WORDS + _VIEW_WORDS * B]
        focal = self._dev[_SEED_WORDS + _VIEW_WORDS * B:_SEED_WORDS + _VIEW_WORDS * B + B]
        cam = self._dev[c0:]
        vm, pm = cam[:16 * B].view(B, 16), cam[16 * B:32 * B].view(B, 16)
        cp, bg = cam[32 * B:35 * B].view(B, 3), cam[35 * B:38 * B].view(B, 3)
        self._upload(settings, *values)
        keep: list = []
        prm = (_lib.Params * B)(*[R._make_params(s._replace(viewmatrix=vm[v], projmatrix=pm[v], campos=cp[v]), P, M,
                                                 keep, dev, bg, v) for v, s in enumerate(settings)])
        table = S._group_table(raw)
        grads = [[torch.zeros_like(t) for t in ts] for ts in raw]
        garr = (_lib.GroupGrad * ng)()
        for k, ts in enumerate(grads):
            for name, t in zip(("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest"), ts):
                setattr(garr[k], name, t.data_ptr() if t.numel() else None)
        self._grad_of = {id(t): g for t, g in zip(flat, [g for gs in grads for g in gs])}
        records = self._adam_records()
        self._scalars = torch.zeros(max(len(records), 1), 6, dtype=torch.float32, device=dev)
        tables = []
        for i0 in range(0, len(records), _lib.ADAM_MAX_TENSORS):
            part = records[i0:i0 + _lib.ADAM_MAX_TENSORS]
            tables.append((i0, (_lib.AdamTensor * len(part))(*[_lib.AdamTensor(p.data_ptr(), g.data_ptr(), m.data_ptr(),
                                                                               v.data_ptr(), p.numel())
                                                                for p, g, m, v, *_ in part])))
        # static outputs and gradient inputs
        color = torch.empty(3, Hs, W, device=dev)
        da = torch.empty(2, Hs, W, device=dev)
        radii = torch.zeros(B, P, dtype=torch.int32, device=dev)
        scales = torch.zeros(B, P, 3, device=dev)
        da4 = torch.zeros(B, 2, H, W, device=dev)
        image, disp, alpha = (torch.zeros(B, 3, H, W, device=dev), torch.zeros(B, 1, H, W, device=dev),
                              torch.zeros(B, 1, H, W, device=dev))
        stats = torch.zeros(B, 8, dtype=torch.int32, device=dev)
        stats_bwd = torch.zeros_like(stats)
        g_image, g_disp, g_alpha = torch.zeros_like(image), torch.zeros_like(disp), torch.zeros_like(alpha)
        g_scales = torch.zeros_like(scales)
        g_color, g_da = torch.zeros(3, Hs, W, device=dev), torch.zeros(2, Hs, W, device=dev)
        d_da4 = torch.zeros_like(da4)
        d_means2D = torch.zeros(B, P, 3, device=dev)
        if self._report is None or self._report.device != dev:
            self._report = torch.zeros(2, dtype=torch.int32, device=dev)
        report = self._report           # one per StepGraph: a re-capture keeps the counts check() has not read yet
        d = R._device_state(dev)
        skey = ("step_graph", id(self))
        if self._scratch_key != (skey, dev):        # this instance's scratch leaves the device state with it
            weakref.finalize(self, d.scratch.pop, skey, None)
            self._scratch_key = (skey, dev)
        fwd_flags = _lib.FWD_DETERMINISTIC if det else 0
        bwd_flags = _lib.BWD_DETERMINISTIC if det else 0
        views_p, seed_p = ptr(views_t), ptr(seed_t)

        def launch(cap, flags, scratch, saved, notify_ptr, seq):
            return lib.b200gsr_forward_scene_dyn(B, prm, ng, table, views_p, seed_p, ptr(scales), ptr(color), ptr(da),
                                                 ptr(radii), ptr(scratch), scratch.numel(), ptr(saved), saved.numel(),
                                                 cap, flags, notify_ptr, seq, _lib.stream(dev))

        def render(saved):
            da4.copy_(da.view(2, B, Hp, W)[:, :, :H].permute(1, 0, 2, 3))
            image.copy_(color.view(3, B, Hp, W)[:, :, :H].permute(1, 0, 2, 3))
            _lib.check(lib.b200gsr_disparity_forward(B, H * W, ptr(da4), ptr(focal), ptr(disp), ptr(stats),
                                                     _lib.stream(dev)), "b200gsr_disparity_forward")
            alpha.copy_(da4[:, 1:2])

        def backward(saved, cap):
            g_color.view(3, B, Hp, W)[:, :, :H].copy_(g_image.permute(1, 0, 2, 3))
            stats_bwd.copy_(stats)
            _lib.check(lib.b200gsr_disparity_backward_ex(B, H * W, ptr(da4), ptr(focal), ptr(g_disp), ptr(g_alpha),
                                                         ptr(stats_bwd), ptr(d_da4), bwd_flags, _lib.stream(dev)),
                       "b200gsr_disparity_backward")
            g_da.view(2, B, Hp, W)[:, :, :H].copy_(d_da4.permute(1, 0, 2, 3))
            _lib.check(lib.b200gsr_backward_scene_dyn(B, prm, ng, table, garr, views_p, seed_p, ptr(g_scales),
                                                      ptr(radii), ptr(da), ptr(g_color), ptr(g_da), ptr(saved),
                                                      saved.numel(), cap, ptr(d_means2D), bwd_flags, _lib.stream(dev)),
                       "b200gsr_backward_scene_dyn")

        layout = (B * P, Hs, W, True, det)
        with torch.no_grad(), torch.cuda.device(dev):
            # eager: measure the pair count synchronously (re-issued with room for it if it overflowed) and run every
            # library path once before capture; nothing is left pending on the device state
            key = (B, P, H, W)
            run_cap, _ = d.capacity_for(key, B * P, False)
            issued = {}

            def issue(c):
                issued["saved"], slot, seq = R._issue_once(d, layout, fwd_flags, c, launch, skey, False,
                                                           "b200gsr_forward_scene_dyn", Exception)
                return slot, seq

            run_cap = d.settle(key, run_cap, *issue(run_cap), issue)
            render(issued["saved"])
            backward(issued["saved"], run_cap)
            # the graphs run at the capacity a later eager forward of this shape would use: the user's, or twice the
            # measured count
            cap = max(run_cap, d.capacity_for(key, B * P, True)[0])
            scratch_bytes, _ = R._layouts(B * P, Hs, W, cap, True, det)
            d.ensure_scratch(skey, scratch_bytes)
            torch.cuda.current_stream(dev).synchronize()
            pool = torch.cuda.graph_pool_handle()
            g_render, g_update = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(g_render, pool=pool):
                saved, _, _ = R._issue_once(d, layout, fwd_flags, cap, launch, skey, True,
                                            "b200gsr_forward_scene_dyn", Exception)
                _lib.check(lib.b200gsr_pair_report(ptr(saved), ptr(report), _lib.stream(dev)), "b200gsr_pair_report")
                render(saved)
            with torch.cuda.graph(g_update, pool=pool):
                backward(saved, cap)
                for i0, arr in tables:
                    _lib.check(lib.b200gsr_adam_step_dyn(len(arr), arr, C.c_void_p(self._scalars.data_ptr() + 24 * i0),
                                                         _lib.stream(dev)), "b200gsr_adam_step_dyn")
        for t in (image, disp, alpha, scales):
            t.requires_grad_(True)
        self._graphs = (g_render, g_update)
        self._keep = (keep, prm, table, garr, tables, raw, saved, color, da, da4, stats, stats_bwd, g_color, g_da, d_da4)
        self._static_grads = (g_image, g_disp, g_alpha, g_scales)
        self._leaves = list(flat)
        self.grads = [dict(zip(S._FIELDS, gs)) for gs in grads]
        self.out = StepOutputs(image, disp, alpha, radii, scales)
        self.d_means2D = d_means2D
        self._cap = cap
        self._key = self._layout(flat, P, M, settings, det)      # after _adam_records created any missing state

    # ---- the step ------------------------------------------------------------------------------------------------
    def render(self, settings_list: Sequence, *, shs_aug=True, scale_aug=True, seed: int | None = None,
               generator: torch.Generator | None = None, focal=None) -> StepOutputs:
        """Replay the render graph for this step's cameras and values (as render_scene + disparity_from_depth_alpha
        on the stacked views).  focal: B floats, default 1 / (2 tanfovx) per view."""
        from . import parallel
        if parallel.reduction_active():
            raise RuntimeError("StepGraph does not reduce gradients over ranks; view sharding cannot be replayed")
        flat, M, P = S._scene_groups(self.groups)
        S._check_device(flat)
        rec = self._views(settings_list, shs_aug, scale_aug, M)
        if seed is None:
            cpu_gen = generator if generator is not None and generator.device.type == "cpu" else None
            seed = int(torch.randint(0, 2 ** 62, (1,), generator=cpu_gen).item())
        if focal is None:
            focal = [1.0 / (2.0 * float(s.tanfovx)) for s in settings_list]
        if len(focal) != self.B:
            raise ValueError(f"StepGraph: expected {self.B} focal lengths")
        det = R.deterministic_mode()
        if self._key is None or self._layout(flat, P, M, settings_list, det) != self._key:
            self._capture(flat, P, M, settings_list, det, (rec, seed, focal))
        else:
            self._upload(settings_list, rec, seed, focal)
        self._graphs[0].replay()
        for t in (self.out.image, self.out.disp, self.out.alpha, self.out.scales):
            t.grad = None
        return self.out

    def step(self) -> None:
        """Replay the update graph: the render backward with the .grad of image / disp / alpha / scales (a missing
        grad counts as zeros), the disparity backward and every optimizer's step.  The leaf gradients come from out.*
        only: a leaf that holds a .grad of its own (a loss term that reaches it directly, or a gradient not cleared
        since an eager step) is refused rather than dropped.  Afterwards `grads` holds the leaf gradients and
        d_means2D the per-view screen-space gradients."""
        if self._key is None:
            raise RuntimeError("StepGraph.step() needs a render() first")
        for t in self._leaves:
            if t.grad is not None:
                raise RuntimeError("StepGraph.step(): a group leaf has a .grad of its own; the update graph computes "
                                   "the leaf gradients from out.image / disp / alpha / scales only and would discard "
                                   "it. Clear the leaves' gradients (optimizer.zero_grad()) and route every loss term "
                                   "through the outputs")
        for t, g in zip((self.out.image, self.out.disp, self.out.alpha, self.out.scales), self._static_grads):
            if t.grad is None:
                g.zero_()
            else:
                g.copy_(t.grad)
            t.grad = None
        records = self._adam_records()      # this step's lr / betas / eps; same tensors as at capture (the layout)
        if records:
            torch._foreach_add_([r[8] for r in records], O._ONE, alpha=1.0)   # as GaussianAdam.step(): counters first
            stage = torch.tensor([O.adam_scalars(lr, b1, b2, eps, st.item())
                                  for _, _, _, _, lr, b1, b2, eps, st in records], dtype=torch.float32).pin_memory()
            self._scalars[:len(records)].copy_(stage, non_blocking=True)
        self._graphs[1].replay()

    def check(self) -> None:
        """Raise PairCapacityOverflow if a render replayed since the last check - under this capture or an earlier
        one - produced more (tile, Gaussian) pairs than its key buffer held (that step's images and gradients are
        invalid).  The capacity is raised and the next render() re-captures.  Waits for the device."""
        if self._report is None:
            return
        rep = self._report.cpu()
        pairs, overflows = int(rep[0]) & 0xFFFFFFFF, int(rep[1])
        if overflows:
            self._report.zero_()
            d = R._device_state(self._report.device)
            d.note((self.B, self.out.radii.shape[1], self.H, self.W), pairs)
            d.grow(pairs)
            self._key = None
            raise R.PairCapacityOverflow(
                f"StepGraph: {overflows} replayed render(s) produced more (tile, Gaussian) pairs than their captured "
                f"key buffer held (up to {pairs}; the current capture holds {self._cap}); their images/gradients are "
                "invalid. The next render() re-captures with room for the count.")
