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

Target mode (the refine stages' reconstruction step, f9) puts the loss into the render graph as well:

    sg = StepGraph(groups, optimizers, views=1, height=H, width=W, target=gt, target_weight=100.0)   # gt [G,3,H,W]
    sg.render(settings_list, shs_aug=False, scale_aug=False, target_index=[i])   # render + recon_l2 loss + gradient
    sg.step()       # no eager loss, no .grad hand-off; sg.loss [B] holds each view's loss

Regulariser mode (the guidance stages' step, f10) puts the reference's total-variation and scale regularisers into the
graphs, so that the eager loss is the guidance term alone:

    sg = StepGraph(groups, optimizers, views=B, height=H, width=W, tv_weight=1.0, tv_depth_weight=1.0,
                   scale_weight=1.0)
    out = sg.render(settings_list, ...)       # also sg.reg_loss [3] = tv(image), tv(disp), mean(mean(scales, -1))
    guidance_loss(out.image).backward()       # eager
    sg.step()       # adds weight * each regulariser's gradient to the outputs' gradients before the render backward

Frozen groups (the scene stages that train one group, f11) are rendered but get no gradient:

    sg = StepGraph(groups, [env_optimizer], views=B, height=H, width=W, frozen=[k != "env" for k in names])

the backward graph computes and stores gradients for the trainable groups only (``grads[k]`` is None for a frozen
group, whose optimizer must not be passed).

Densification statistics (f12): the reference's add_densification_stats of the step's last view, gathered inside the
backward graph instead of by an eager kernel over ``d_means2D`` afterwards:

    sg = StepGraph(groups, optimizers, views=B, height=H, width=W,
                   densify_stats=[(g.xyz_gradient_accum, g.denom, g.max_radii2D) for g in models], keep_means2D=False)
    sg.step(stats_view=-1 if step < densify_until_iter else None)     # -1 = view B-1, None = off; no re-capture

Reserved groups (f13, dreamscene_b200.reserve.ReservedGroup) hold their rows at a fixed capacity with the live count
in device memory, so densify, prune, filter and opacity reset rewrite a prefix of the same tensors and the next
render() replays instead of capturing again:

    g = ReservedGroup.from_group(model)
    sg = StepGraph([g], [opt], views=B, height=H, width=W, densify_stats=[g], keep_means2D=False)
    out = sg.render(...); loss.backward(); sg.step(optimize=False, stats_view=-1)
    g.densify_and_prune(opt, max_grad, min_opacity, extent, max_screen_size)     # the next render() replays

Reserved and plain groups mix (a plain group's live count is its row count).  The layout holds the capacities;
out.radii, out.scales, d_means2D and grads keep the capacity layout with zeros in the dead rows.  A densify_stats
entry may be the reserved group itself (its statistics, followed through a growth).

``step(optimize=False)`` replays the backward only (``grads`` and ``d_means2D``), leaving parameters, moments and
step counters as they are: the reference's densify step, whose optimizer.step() follows densify_and_prune and so
updates nothing.

The first ``render()`` of a layout runs one eager forward and backward (which measure the pair capacity and set up
the library) and then captures.  The layout - P, the group tensors, the optimizer state tensors, the per-view
scale_modifier, deterministic mode, the target tensor and weight, the regulariser weights, the frozen groups and the
densification statistics tensors - is compared on the host at every ``render()``; a change (densify / prune, or
assigning ``frozen`` / ``densify_stats``) re-captures.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import NamedTuple, Sequence

import torch

from . import _lib
from . import optim as O
from . import rasterizer as R
from . import reserve as RS
from . import scene as S

_SEED_WORDS = 8             # the uint64 seed, padded so the view records start 32-byte aligned
_VIEW_WORDS = 8             # sizeof(b200gsr_step_view) / 4


class StepOutputs(NamedTuple):
    """Static tensors, overwritten by the next render().  image / disp / alpha / scales are leaves that require grad
    (except in target mode): the loss's gradients reach step() through their .grad."""
    image: torch.Tensor     # [B,3,H,W]
    disp: torch.Tensor      # [B,1,H,W]
    alpha: torch.Tensor     # [B,1,H,W]
    radii: torch.Tensor     # [B,P] int32
    scales: torch.Tensor    # [B,P,3] the augmented scales (for the scale loss)


class StepGraph:
    """One training step of `views` views of height x width over the parameter groups `groups` (as render_scene),
    with the GaussianAdam optimizers `optimizers` over their leaves, replayed from CUDA graphs.

    target: a CUDA [G,3,H,W] float16 / float32 contiguous tensor of pseudo ground truths, read in place at every
    replay.  The render graph then also computes view v's loss target_weight * mean((fp16(image_v) - target[i_v])^2)
    (dreamscene_b200.losses.recon_l2_loss) into `loss` and its image gradient; the step minimises the views' sum.

    tv_weight / tv_depth_weight / scale_weight: the weights of the reference's regularisers tv_loss(image),
    tv_loss(disp) and mean(mean(scales, -1)) (dreamscene_b200.losses.tv_loss), computed inside the graphs.  A term
    whose weight is None or 0 is off.  The render graph writes the unweighted values into `reg_loss`; the backward
    graph adds weight * each term's gradient to the gradient step() takes from the output's .grad, which is the
    eager step's gradient bit for bit when the eager loss, written before the regularisers, reaches each output
    through one edge.  Not with target (the refine stages use no regulariser).

    frozen: None, or one bool per group (render_scene's `frozen`).  A frozen group is rendered but its leaves get no
    gradient buffer (grads[k] is None) and the backward does no work for it; an optimizer over one of its leaves is
    refused.  The regularisers are unchanged: the scale term still covers every group's rows.  Assigning
    `sg.frozen` re-captures at the next render().

    densify_stats: None, or one entry per group (render_scene's `densify_stats`): None, or the group's
    (xyz_gradient_accum, denom, max_radii2D or None), updated in place by the backward graph for the view that step()
    selects.  Their pointers are part of the layout: densify / prune replaces them together with the leaves, and
    assigning the new ones to `sg.densify_stats` re-captures at the next render().  A frozen group's entry is refused.

    keep_means2D: False leaves `d_means2D` None: the backward stores no [B,P,3] screen-space gradient (the statistics
    need none).  True (default) keeps it."""

    def __init__(self, groups: Sequence, optimizers: Sequence, *, views: int, height: int, width: int,
                 target: torch.Tensor | None = None, target_weight: float = 100.0, tv_weight: float | None = None,
                 tv_depth_weight: float | None = None, scale_weight: float | None = None,
                 frozen: Sequence[bool] | None = None, densify_stats: Sequence | None = None,
                 keep_means2D: bool = True):
        self.groups = list(groups)
        self.optimizers = list(optimizers)
        self.B, self.H, self.W = int(views), int(height), int(width)
        if not 1 <= self.B <= _lib.MAX_VIEWS:
            raise ValueError(f"StepGraph: views must be in 1..{_lib.MAX_VIEWS}")
        for opt in self.optimizers:
            if not isinstance(opt, O.GaussianAdam):
                raise TypeError(f"StepGraph: only GaussianAdam optimizers can be replayed, got {type(opt).__name__}")
        self.target, self.target_weight = target, float(target_weight)
        self._target_key()
        self.tv_weight, self.tv_depth_weight, self.scale_weight = tv_weight, tv_depth_weight, scale_weight
        self._reg_key()
        self.frozen = frozen
        self._frozen_key()
        self.densify_stats = densify_stats
        self.keep_means2D = bool(keep_means2D)
        self._stats_key()
        self._key = None
        self._report = None         # device [2]: max pair count, overflowed replays; kept across re-captures
        self._scratch_key = None
        self._stats_view = None     # with densify_stats: (device int32 [1] read by the backward graph, its value)
        self.d_means2D = None       # [B,P,3] per-view screen-space gradients of the last step (None: keep_means2D=False)
        self.grads = None           # per group {leaf name: its gradient of the last step} (the backward graph's buffers),
                                    # None for a frozen group
        self.loss = None            # target mode: [B] each view's loss of the last render(), in the target's dtype
        self.reg_loss = None        # with a regulariser: [3] float32 tv(image), tv(disp), scale of the last render()

    def _target_key(self):
        """Host checks of `target` (its device is checked in render()) -> its part of the layout key, None without."""
        t = self.target
        if t is None:
            return None
        if not torch.is_tensor(t) or t.dtype not in (torch.float16, torch.float32):
            raise TypeError("StepGraph: target must be a float16 or float32 tensor")
        if t.dim() != 4 or t.shape[0] < 1 or tuple(t.shape[1:]) != (3, self.H, self.W):
            raise ValueError(f"StepGraph: target must be [G,3,{self.H},{self.W}] with G >= 1, got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise ValueError("StepGraph: target must be contiguous (it is read in place at every replay)")
        if 3 * self.H * self.W >= 2 ** 31:
            raise ValueError("StepGraph: target mode needs 3 H W < 2^31")
        return t.data_ptr(), t.dtype, tuple(t.shape), self.target_weight

    def _reg_key(self):
        """Host checks of the regulariser weights -> the weights of the terms that are on (tv(image), tv(disp),
        scale; None for a term that is off), part of the layout key."""
        out = []
        for name in ("tv_weight", "tv_depth_weight", "scale_weight"):
            w = getattr(self, name)
            if w is not None:
                w = float(w)
                if not (0.0 <= w < float("inf")):
                    raise ValueError(f"StepGraph: {name} must be finite and >= 0, got {w}")
            out.append(w if w else None)
        if any(w is not None for w in out):
            if self.target is not None:
                raise ValueError("StepGraph: the regularisers (tv_weight, tv_depth_weight, scale_weight) cannot be "
                                 "combined with target=")
            if (out[0] is not None or out[1] is not None) and (self.H < 2 or self.W < 2):
                raise ValueError("StepGraph: the total-variation regularisers need height and width >= 2")
        return tuple(out)

    def _frozen_key(self) -> int:
        """The frozen groups' bit mask (bit g = group g), part of the layout key."""
        return S._frozen_mask(self.frozen, len(self.groups), "StepGraph")

    def _stats(self):
        """The validated densify_stats entries (scene._densify_stats), None when no group gathers.  An entry that is a
        ReservedGroup stands for its current statistics tensors."""
        entries = self.densify_stats
        if entries is not None:
            entries = [e.stats if isinstance(e, RS.ReservedGroup) else e for e in entries]
        return S._densify_stats(entries, self.groups, self._frozen_key(), "StepGraph")

    def _reserved(self):
        """One bool per group: a ReservedGroup (part of the layout key: it selects the _live entry points)."""
        return tuple(isinstance(g, RS.ReservedGroup) for g in self.groups)

    def _stats_key(self):
        """The statistics tensors' pointers and keep_means2D, part of the layout key."""
        st = self._stats()
        ptrs = None if st is None else tuple(None if e is None else tuple(0 if t is None else t.data_ptr() for t in e)
                                             for e in st)
        return ptrs, bool(self.keep_means2D)

    def _check_frozen_leaves(self, flat, mask):
        """Refuse an optimizer parameter that is a leaf of a frozen group: it would never get a gradient."""
        frozen = {id(t): i // 6 for i, t in enumerate(flat) if (mask >> (i // 6)) & 1}
        for opt in self.optimizers:
            for group in opt.param_groups:
                for p in group["params"]:
                    if id(p) in frozen:
                        raise ValueError(f"StepGraph: an optimizer parameter is a leaf of frozen group {frozen[id(p)]}; "
                                         "it would never get a gradient. Leave that group's optimizer out or unfreeze "
                                         "the group")

    def _target_indices(self, target_index):
        """-> the B validated target indices, or None without a target."""
        if self._target_key() is None:
            if target_index is not None:
                raise ValueError("StepGraph: target_index needs a StepGraph built with target=")
            return None
        if target_index is None:
            raise ValueError("StepGraph: a StepGraph with a target needs render(..., target_index=[one per view])")
        idx = [int(i) for i in target_index]
        G = int(self.target.shape[0])
        if len(idx) != self.B:
            raise ValueError(f"StepGraph: expected {self.B} target indices, got {len(idx)}")
        if not all(0 <= i < G for i in idx):
            raise ValueError(f"StepGraph: target indices must be in 0..{G - 1}, got {idx}")
        return idx

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
        return (P, M, ptrs, tuple(states), tuple(float(s.scale_modifier) for s in settings), det, self._target_key(),
                self._reg_key(), self._frozen_key(), self._stats_key(), self._reserved())

    def _upload(self, settings, rec, seed, focal, tidx):
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
        stage[f0 + B:f0 + 2 * B].view(torch.int32)[:] = torch.tensor(tidx or [0] * B, dtype=torch.int32)
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
        """Allocate the static buffers, upload this step's `values` = (records, seed, focal, target indices), run the
        step's render and backward eagerly once (measuring the pair capacity), then capture the render, backward and
        Adam graphs."""
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
        f0 = _SEED_WORDS + _VIEW_WORDS * B
        self._cam0 = c0 = (f0 + 2 * B + 63) // 64 * 64
        # [seed | B view records | B focal lengths | B target indices | pad | B viewmatrix, B projmatrix, B campos, B bg]
        self._dev = torch.zeros(c0 + B * 38, dtype=torch.float32, device=dev)
        seed_t = self._dev[:2].view(torch.int64)
        views_t = self._dev[_SEED_WORDS:f0]
        focal = self._dev[f0:f0 + B]
        tidx_t = self._dev[f0 + B:f0 + 2 * B].view(torch.int32)
        cam = self._dev[c0:]
        vm, pm = cam[:16 * B].view(B, 16), cam[16 * B:32 * B].view(B, 16)
        cp, bg = cam[32 * B:35 * B].view(B, 3), cam[35 * B:38 * B].view(B, 3)
        self._upload(settings, *values)
        keep: list = []
        prm = (_lib.Params * B)(*[R._make_params(s._replace(viewmatrix=vm[v], projmatrix=pm[v], campos=cp[v]), P, M,
                                                 keep, dev, bg, v) for v, s in enumerate(settings)])
        table = S._group_table(raw)
        fmask = self._frozen_key()
        grads = [[None] * 6 if (fmask >> k) & 1 else [torch.zeros_like(t) for t in ts] for k, ts in enumerate(raw)]
        # reserved groups: the live row counts the kernels read, copied from each group's `live` at the start of
        # every render (a plain group's entry is its row count)
        reserved = self._reserved()
        live_mode = any(reserved)
        live_t = torch.tensor([int(ts[0].shape[0]) for ts in raw], dtype=torch.int32, device=dev)
        group_of = {id(t): i // 6 for i, t in enumerate(flat)}

        def copy_live():
            for k, g in enumerate(self.groups):
                if reserved[k]:
                    live_t[k:k + 1].copy_(g.live)
        garr = (_lib.GroupGrad * ng)()
        for k, ts in enumerate(grads):
            for name, t in zip(("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest"), ts):
                setattr(garr[k], name, t.data_ptr() if t is not None and t.numel() else None)
        self._grad_of = {id(t): g for t, g in zip(flat, [g for gs in grads for g in gs]) if g is not None}
        records = self._adam_records()
        self._scalars = torch.zeros(max(len(records), 1), 6, dtype=torch.float32, device=dev)
        tables = []
        for i0 in range(0, len(records), _lib.ADAM_MAX_TENSORS):
            part = records[i0:i0 + _lib.ADAM_MAX_TENSORS]
            live_arr = None
            if live_mode:       # each reserved leaf stops at its group's live rows
                live_arr = (_lib.AdamLive * len(part))(*[
                    _lib.AdamLive(live_t.data_ptr() + 4 * group_of[id(p)], p[0].numel() if p.shape[0] else 1, 0)
                    if reserved[group_of[id(p)]] else _lib.AdamLive(None, 0, 0) for p, *_ in part])
            tables.append((i0, (_lib.AdamTensor * len(part))(*[_lib.AdamTensor(p.data_ptr(), g.data_ptr(), m.data_ptr(),
                                                                               v.data_ptr(), p.numel())
                                                                for p, g, m, v, *_ in part]), live_arr))
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
        d_means2D = torch.zeros(B, P, 3, device=dev) if self.keep_means2D else None
        dstats = self._stats()
        # the backward with the statistics entry point when it gathers or stores no d_means2D; its view is read from
        # stats_view_t at every replay (step() writes it; -1 = off, as for the eager run below)
        with_stats = dstats is not None or d_means2D is None
        stats_view_t = torch.full((1,), -1, dtype=torch.int32, device=dev)
        stats_arr = S._stats_table(dstats)
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
        target = self.target
        loss = None
        if target is not None:
            # the views' loss and its image gradient into g_image, for an incoming gradient of 1 per view
            loss = torch.zeros(B, dtype=target.dtype, device=dev)
            ones = torch.ones(B, dtype=target.dtype, device=dev)
            l2_scratch = torch.empty(lib.b200gsr_recon_l2_scratch_bytes(B, 3 * H * W), dtype=torch.uint8, device=dev)
            keep.append((ones, l2_scratch))
        reg = self._reg_key()
        reg_loss = None
        if any(w is not None for w in reg):
            # each term's value into reg_loss, and weight * its gradient added to the output's gradient buffer
            reg_loss = torch.zeros(3, dtype=torch.float32, device=dev)
            reg_go = torch.tensor([w or 0.0 for w in reg], dtype=torch.float32, device=dev)
            tv_scratch = [torch.empty(lib.b200gsr_tv_loss_scratch_bytes(B, c, H, W), dtype=torch.uint8, device=dev)
                          for c in (3, 1)]
            scale_scratch = torch.empty(lib.b200gsr_scale_loss_scratch_bytes(B * P), dtype=torch.uint8, device=dev)
            keep.append((reg_go, tv_scratch, scale_scratch))

        def regularisers(forward, scale_acc=1):
            for k, (x, c, gx) in enumerate(((image, 3, g_image), (disp, 1, g_disp))):
                if reg[k] is not None:
                    _lib.check(lib.b200gsr_tv_loss(B, c, H, W, ptr(x), None if forward else ptr(reg_go[k]),
                                                   ptr(reg_loss[k]) if forward else None, None if forward else ptr(gx),
                                                   1, ptr(tv_scratch[k]), tv_scratch[k].numel(), _lib.stream(dev)),
                               "b200gsr_tv_loss")
            if reg[2] is not None and live_mode:        # the mean over the live rows
                _lib.check(lib.b200gsr_scale_loss_live(B, ng, table, ptr(live_t), ptr(scales),
                                                       None if forward else ptr(reg_go[2]),
                                                       ptr(reg_loss[2]) if forward else None,
                                                       None if forward else ptr(g_scales), scale_acc, ptr(scale_scratch),
                                                       scale_scratch.numel(), _lib.stream(dev)),
                           "b200gsr_scale_loss_live")
            elif reg[2] is not None:
                _lib.check(lib.b200gsr_scale_loss(B * P, ptr(scales), None if forward else ptr(reg_go[2]),
                                                  ptr(reg_loss[2]) if forward else None,
                                                  None if forward else ptr(g_scales), scale_acc, ptr(scale_scratch),
                                                  scale_scratch.numel(), _lib.stream(dev)), "b200gsr_scale_loss")

        def launch(cap, flags, scratch, saved, notify_ptr, seq):
            if live_mode:
                return lib.b200gsr_forward_scene_dyn_live(B, prm, ng, table, views_p, seed_p, ptr(scales), ptr(color),
                                                          ptr(da), ptr(radii), ptr(scratch), scratch.numel(), ptr(saved),
                                                          saved.numel(), cap, flags, notify_ptr, seq, ptr(live_t),
                                                          _lib.stream(dev))
            return lib.b200gsr_forward_scene_dyn(B, prm, ng, table, views_p, seed_p, ptr(scales), ptr(color), ptr(da),
                                                 ptr(radii), ptr(scratch), scratch.numel(), ptr(saved), saved.numel(),
                                                 cap, flags, notify_ptr, seq, _lib.stream(dev))

        def render(saved):
            da4.copy_(da.view(2, B, Hp, W)[:, :, :H].permute(1, 0, 2, 3))
            image.copy_(color.view(3, B, Hp, W)[:, :, :H].permute(1, 0, 2, 3))
            _lib.check(lib.b200gsr_disparity_forward(B, H * W, ptr(da4), ptr(focal), ptr(disp), ptr(stats),
                                                     _lib.stream(dev)), "b200gsr_disparity_forward")
            alpha.copy_(da4[:, 1:2])
            if target is not None:
                _lib.check(lib.b200gsr_recon_l2(B, 3 * H * W, ptr(image), ptr(target),
                                                int(target.dtype == torch.float16), target.shape[0], ptr(tidx_t),
                                                self.target_weight, ptr(ones), ptr(loss), ptr(g_image),
                                                ptr(l2_scratch), l2_scratch.numel(), _lib.stream(dev)),
                           "b200gsr_recon_l2")
            if reg_loss is not None:
                regularisers(True)

        def backward(saved, cap, scale_acc=1):
            if reg_loss is not None:
                regularisers(False, scale_acc)
            g_color.view(3, B, Hp, W)[:, :, :H].copy_(g_image.permute(1, 0, 2, 3))
            stats_bwd.copy_(stats)
            _lib.check(lib.b200gsr_disparity_backward_ex(B, H * W, ptr(da4), ptr(focal), ptr(g_disp), ptr(g_alpha),
                                                         ptr(stats_bwd), ptr(d_da4), bwd_flags, _lib.stream(dev)),
                       "b200gsr_disparity_backward")
            g_da.view(2, B, Hp, W)[:, :, :H].copy_(d_da4.permute(1, 0, 2, 3))
            if live_mode:
                _lib.check(lib.b200gsr_backward_scene_dyn_live(B, prm, ng, table, garr, views_p, seed_p, ptr(g_scales),
                                                               ptr(radii), ptr(da), ptr(g_color), ptr(g_da), ptr(saved),
                                                               saved.numel(), cap, ptr(d_means2D), bwd_flags, fmask,
                                                               stats_arr, ptr(stats_view_t), ptr(live_t),
                                                               _lib.stream(dev)),
                           "b200gsr_backward_scene_dyn_live")
                return
            if with_stats:
                _lib.check(lib.b200gsr_backward_scene_dyn_stats(B, prm, ng, table, garr, views_p, seed_p, ptr(g_scales),
                                                                ptr(radii), ptr(da), ptr(g_color), ptr(g_da), ptr(saved),
                                                                saved.numel(), cap, ptr(d_means2D), bwd_flags, fmask,
                                                                stats_arr, ptr(stats_view_t), _lib.stream(dev)),
                           "b200gsr_backward_scene_dyn_stats")
                return
            _lib.check(lib.b200gsr_backward_scene_dyn_frozen(B, prm, ng, table, garr, views_p, seed_p, ptr(g_scales),
                                                             ptr(radii), ptr(da), ptr(g_color), ptr(g_da), ptr(saved),
                                                             saved.numel(), cap, ptr(d_means2D), bwd_flags, fmask,
                                                             _lib.stream(dev)),
                       "b200gsr_backward_scene_dyn_frozen")

        layout = (B * P, Hs, W, True, det)
        with torch.no_grad(), torch.cuda.device(dev):
            # eager: measure the pair count synchronously (re-issued with room for it if it overflowed) and run every
            # library path once before capture; nothing is left pending on the device state
            key = (B, P, H, W)
            run_cap, _ = d.capacity_for(key, B * P, False)
            issued = {}
            copy_live()

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
            if live_mode:
                # reserved rows: the measured pairs per live row (with the 2x head-room of d.note) for every row of the
                # capacity, so that an event that fills the reserve replays without overflowing (DESIGN.md f13)
                p_live = sum(g.live_count if reserved[k] else int(raw[k][0].shape[0]) for k, g in enumerate(self.groups))
                if p_live > 0:
                    cap = max(cap, R._round_cap(-(-d.caps.get(key, cap) * P // p_live)))
            scratch_bytes, _ = R._layouts(B * P, Hs, W, cap, True, det)
            d.ensure_scratch(skey, scratch_bytes)
            torch.cuda.current_stream(dev).synchronize()
            pool = torch.cuda.graph_pool_handle()
            g_render, g_backward = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            g_adam = torch.cuda.CUDAGraph() if tables else None     # an empty graph cannot be replayed
            with torch.cuda.graph(g_render, pool=pool):
                copy_live()
                saved, _, _ = R._issue_once(d, layout, fwd_flags, cap, launch, skey, True,
                                            "b200gsr_forward_scene_dyn", Exception)
                _lib.check(lib.b200gsr_pair_report(ptr(saved), ptr(report), _lib.stream(dev)), "b200gsr_pair_report")
                render(saved)
            with torch.cuda.graph(g_backward, pool=pool):
                backward(saved, cap)
            # with the scale regulariser, a second backward graph that writes its constant gradient into g_scales
            # instead of adding it, for steps whose loss leaves out.scales without a .grad (the guidance stages'
            # usual case): it saves a fill and a read of the [B,P,3] buffer
            g_backward_w = None
            if reg[2] is not None:
                g_backward_w = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g_backward_w, pool=pool):
                    backward(saved, cap, scale_acc=0)
            if g_adam is not None:
                with torch.cuda.graph(g_adam, pool=pool):
                    for i0, arr, live_arr in tables:
                        scal = C.c_void_p(self._scalars.data_ptr() + 24 * i0)
                        if live_arr is not None:
                            _lib.check(lib.b200gsr_adam_step_dyn_live(len(arr), arr, scal, live_arr, _lib.stream(dev)),
                                       "b200gsr_adam_step_dyn_live")
                        else:
                            _lib.check(lib.b200gsr_adam_step_dyn(len(arr), arr, scal, _lib.stream(dev)),
                                       "b200gsr_adam_step_dyn")
        if target is None:
            for t in (image, disp, alpha, scales):
                t.requires_grad_(True)
        self._graphs = (g_render, g_backward, g_adam, g_backward_w)
        self.loss = loss
        self.reg_loss = reg_loss
        self._accumulated = [reg[0] is not None, reg[1] is not None, False, reg[2] is not None]
        self._keep = (keep, prm, table, garr, tables, raw, saved, color, da, da4, stats, stats_bwd, g_color, g_da, d_da4,
                      stats_arr, stats_view_t, live_t)
        self._stats_view = (stats_view_t, -1) if dstats is not None else None    # device slot, value last written
        self._static_grads = (g_image, g_disp, g_alpha, g_scales)
        self._leaves = list(flat)
        self.grads = [None if gs[0] is None else dict(zip(S._FIELDS, gs)) for gs in grads]
        self.out = StepOutputs(image, disp, alpha, radii, scales)
        self.d_means2D = d_means2D
        self._cap = cap
        self._key = self._layout(flat, P, M, settings, det)      # after _adam_records created any missing state

    # ---- the step ------------------------------------------------------------------------------------------------
    def render(self, settings_list: Sequence, *, shs_aug=True, scale_aug=True, seed: int | None = None,
               generator: torch.Generator | None = None, focal=None, target_index=None) -> StepOutputs:
        """Replay the render graph for this step's cameras and values (as render_scene + disparity_from_depth_alpha
        on the stacked views).  focal: B floats, default 1 / (2 tanfovx) per view.  target_index: in target mode (only
        there), B indices into the target, view v's pseudo ground truth; the graph also computes `loss`."""
        from . import parallel
        if parallel.reduction_active():
            raise RuntimeError("StepGraph does not reduce gradients over ranks; view sharding cannot be replayed")
        flat, M, P = S._scene_groups(self.groups)
        S._check_device(flat)
        for k, g in enumerate(self.groups):
            if isinstance(g, RS.ReservedGroup) and not (0 <= g.live_count <= g.capacity and g.live.numel() == 1 and
                                                         g.live.dtype == torch.int32 and g.live.device == flat[0].device):
                raise ValueError(f"StepGraph: reserved group {k}: live count {g.live_count} not in 0..{g.capacity} or "
                                 "its `live` is not a device int32 [1] on the groups' device")
        rec = self._views(settings_list, shs_aug, scale_aug, M)
        tidx = self._target_indices(target_index)
        self._reg_key()
        self._check_frozen_leaves(flat, self._frozen_key())
        self._stats_key()
        if tidx is not None and (self.target.device.type != "cuda" or self.target.device != flat[0].device):
            raise ValueError("StepGraph: target must be a CUDA tensor on the groups' device")
        if seed is None:
            cpu_gen = generator if generator is not None and generator.device.type == "cpu" else None
            seed = int(torch.randint(0, 2 ** 62, (1,), generator=cpu_gen).item())
        if focal is None:
            focal = [1.0 / (2.0 * float(s.tanfovx)) for s in settings_list]
        if len(focal) != self.B:
            raise ValueError(f"StepGraph: expected {self.B} focal lengths")
        det = R.deterministic_mode()
        if self._key is None or self._layout(flat, P, M, settings_list, det) != self._key:
            self._capture(flat, P, M, settings_list, det, (rec, seed, focal, tidx))
        else:
            self._upload(settings_list, rec, seed, focal, tidx)
        self._graphs[0].replay()
        for t in (self.out.image, self.out.disp, self.out.alpha, self.out.scales):
            t.grad = None
        return self.out

    def step(self, optimize: bool = True, stats_view: int | None = -1) -> None:
        """Replay the backward graph: the render backward with the .grad of image / disp / alpha / scales (a missing
        grad counts as zeros; in target mode the loss's image gradient from the render graph instead) plus each
        regulariser's weighted gradient, the disparity backward; then, with `optimize`, the Adam graph: every
        optimizer's step.  The leaf gradients come from out.* only: a leaf that holds a .grad of its own (a loss term
        that reaches it directly, or a gradient not cleared since an eager step) is refused rather than dropped.
        Afterwards `grads` holds the leaf gradients and d_means2D the per-view screen-space gradients.

        stats_view (with densify_stats): the view whose densification statistics this backward adds, -1 = the last
        view (B - 1), or None = none (past the reference's densify_until_iter).  Written to device memory with the
        step's other values: no re-capture.  The statistics are gathered by the backward graph, so optimize=False steps
        gather them too, as the reference's add_densification_stats precedes its densify and optimizer.step().

        optimize=False leaves parameters, moments and step counters untouched, as the reference's optimizer.step()
        after densify_and_prune (whose new leaves have no gradient) does.  A step where only some leaves skip Adam
        (reset_opacity replaces the opacity leaf only) is step(optimize=False) followed by an eager
        GaussianAdam.step() over the others' `grads` (INTEGRATION.md section 4c)."""
        if self._key is None:
            raise RuntimeError("StepGraph.step() needs a render() first")
        for t in self._leaves:
            if t.grad is not None:
                raise RuntimeError("StepGraph.step(): a group leaf has a .grad of its own; the update graph computes "
                                   "the leaf gradients from out.image / disp / alpha / scales only and would discard "
                                   "it. Clear the leaves' gradients (optimizer.zero_grad()) and route every loss term "
                                   "through the outputs")
        # the backward graph that writes the scale regulariser's gradient into g_scales, when there is no eager
        # gradient of out.scales to add it to
        write_scales = self._graphs[3] is not None and self.out.scales.grad is None
        if self.loss is None:
            for t, g, acc in zip((self.out.image, self.out.disp, self.out.alpha, self.out.scales), self._static_grads,
                                 self._accumulated):
                if t.grad is not None:
                    g.copy_(t.grad)
                elif not acc:
                    g.zero_()
                elif not (write_scales and t is self.out.scales):
                    g.fill_(-0.0)       # -0 + r == r bitwise, the sign of zero included: the regulariser's gradient
                t.grad = None
        if stats_view is not None and not -1 <= int(stats_view) < self.B:
            raise ValueError(f"StepGraph.step(): stats_view must be -1 (the last view), None or in 0..{self.B - 1}, "
                             f"got {stats_view}")
        if self._stats_view is not None:
            sv = -1 if stats_view is None else (self.B - 1 if int(stats_view) == -1 else int(stats_view))
            slot, last = self._stats_view
            if sv != last:
                slot.copy_(torch.tensor([sv], dtype=torch.int32).pin_memory(), non_blocking=True)
                self._stats_view = (slot, sv)
        if optimize:
            records = self._adam_records()      # this step's lr / betas / eps; same tensors as at capture (the layout)
            if records:
                torch._foreach_add_([r[8] for r in records], O._ONE, alpha=1.0)   # as GaussianAdam.step(): counters first
                stage = torch.tensor([O.adam_scalars(lr, b1, b2, eps, st.item())
                                      for _, _, _, _, lr, b1, b2, eps, st in records], dtype=torch.float32).pin_memory()
                self._scalars[:len(records)].copy_(stage, non_blocking=True)
        self._graphs[3 if write_scales else 1].replay()
        if optimize and self._graphs[2] is not None:
            self._graphs[2].replay()

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
