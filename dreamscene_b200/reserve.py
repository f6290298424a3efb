"""Parameter groups with reserved rows (DESIGN.md section 0, f13): densify, prune, filter and opacity reset in place,
so that a StepGraph over the group keeps its captured graphs.

A ``ReservedGroup`` allocates its six leaves, their Adam moments and its densification statistics once at a row
capacity.  Rows [0, live_count) are the Gaussians; the rest are absent: the replayed step culls them before reading
them (include/b200gsr_reserve.h), gives them zero gradients and leaves their parameters and moments untouched.  An
event computes its result with the f4 / f5 functions (densify.densify_and_prune, densify.prune_points,
filtering.gaussian_filtering) over the live prefix and copies it back into the prefix of the same tensors, so their
pointers and shapes - the layout a StepGraph captured - stay put:

    g = ReservedGroup.from_group(model)                  # capacity = live * (1 + DEFAULT_HEADROOM)
    opt = GaussianAdam(g.param_groups(lrs), eps=1e-15)
    sg = StepGraph([g], [opt], views=B, height=H, width=W, densify_stats=[g], keep_means2D=False)
    ...
    sg.step(optimize=False, stats_view=-1)
    g.densify_and_prune(opt, max_grad, min_opacity, extent, max_screen_size)   # next sg.render() replays

Only an event whose result exceeds the capacity re-allocates (with headroom again) and moves the optimizer state to
the new tensors; the StepGraph then captures once more.  Eager render_scene refuses a ReservedGroup: render
``g.rows()``, the live prefixes as zero-copy views.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Optional

import torch

from . import densify as D
from . import filtering as F
from .scene import _FIELDS

DEFAULT_HEADROOM = 1.0      # capacity = ceil(live * (1 + headroom)): room for one event that doubles the group
_NAMES = dict(zip(("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest"), _FIELDS))   # densify name -> leaf
_STATS = ("xyz_gradient_accum", "denom", "max_radii2D")


def capacity_for(rows: int, headroom: float = DEFAULT_HEADROOM) -> int:
    """The capacity allocated for `rows` live rows: ceil(rows * (1 + headroom)), at least rows + 1."""
    if not headroom >= 0.0 or math.isinf(headroom):
        raise ValueError(f"ReservedGroup: headroom must be finite and >= 0, got {headroom}")
    return max(int(math.ceil(rows * (1.0 + headroom))), rows + 1)


class ReservedGroup:
    """One Gaussian parameter group at a fixed row capacity: the attributes render_scene / StepGraph read
    (_xyz [cap,3], _opacity [cap,1], _scaling [cap,3], _rotation [cap,4], _features_dc [cap,1,3], _features_rest
    [cap,M-1,3], nn.Parameters), the statistics xyz_gradient_accum [cap,1], denom [cap,1], max_radii2D [cap],
    ``live`` (device int32 [1], read by the replayed step) and ``live_count`` (its host mirror)."""

    _reserved_rows = True       # render_scene refuses the type (it would render the dead rows)

    def __init__(self, leaves: dict, stats: dict, live_count: int, headroom: float = DEFAULT_HEADROOM):
        cap = int(leaves["_xyz"].shape[0])
        for name in _FIELDS:
            t = leaves[name]
            if int(t.shape[0]) != cap:
                raise ValueError(f"ReservedGroup: {name} has {int(t.shape[0])} rows, _xyz has {cap}")
        for name in _STATS:
            if stats[name].numel() != cap:
                raise ValueError(f"ReservedGroup: {name} has {stats[name].numel()} elements, the capacity is {cap}")
        if not 0 <= int(live_count) <= cap:
            raise ValueError(f"ReservedGroup: live count {live_count} not in 0..{cap} (the capacity)")
        for name in _FIELDS:
            setattr(self, name, leaves[name])
        for name in _STATS:
            setattr(self, name, stats[name])
        self.headroom = float(headroom)
        self.live_count = int(live_count)
        self.live = torch.tensor([self.live_count], dtype=torch.int32, device=self._xyz.device)

    # ---- construction ------------------------------------------------------------------------------------------
    @classmethod
    def from_tensors(cls, xyz, features_dc, features_rest, opacity, scaling, rotation, *, capacity: int | None = None,
                     headroom: float = DEFAULT_HEADROOM, stats=None) -> "ReservedGroup":
        """A group holding these rows (copied) at `capacity` rows (default capacity_for(rows, headroom)).  stats:
        optional (xyz_gradient_accum, denom, max_radii2D) of the rows, zeros otherwise.  Dead rows start at zero."""
        n = int(xyz.shape[0])
        cap = capacity_for(n, headroom) if capacity is None else int(capacity)
        if cap < n:
            raise ValueError(f"ReservedGroup: capacity {cap} is below the {n} rows")
        leaves = {}
        for name, t in zip(("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"),
                           (xyz, features_dc, features_rest, opacity, scaling, rotation)):
            full = torch.zeros((cap,) + tuple(t.shape[1:]), dtype=torch.float32, device=t.device)
            full[:n] = t.detach()
            leaves[name] = torch.nn.Parameter(full.requires_grad_(True))
        dev = xyz.device
        st = {"xyz_gradient_accum": torch.zeros(cap, 1, device=dev), "denom": torch.zeros(cap, 1, device=dev),
              "max_radii2D": torch.zeros(cap, device=dev)}
        if stats is not None:
            for name, t in zip(_STATS, stats):
                st[name].view(-1)[:n] = t.detach().reshape(-1)
        return cls(leaves, st, n, headroom)

    @classmethod
    def from_group(cls, g, *, capacity: int | None = None, headroom: float = DEFAULT_HEADROOM) -> "ReservedGroup":
        """from_tensors over a reference GaussianModel's leaves (and its statistics, when it has them)."""
        stats = None
        if all(getattr(g, name, None) is not None for name in _STATS) and \
                all(getattr(g, name).numel() == g._xyz.shape[0] for name in _STATS):
            stats = tuple(getattr(g, name) for name in _STATS)
        return cls.from_tensors(g._xyz, g._features_dc, g._features_rest, g._opacity, g._scaling, g._rotation,
                                capacity=capacity, headroom=headroom, stats=stats)

    # ---- views -------------------------------------------------------------------------------------------------
    @property
    def capacity(self) -> int:
        return int(self._xyz.shape[0])

    @property
    def stats(self):
        """(xyz_gradient_accum, denom, max_radii2D) at capacity: StepGraph's densify_stats entry (or pass the group)."""
        return tuple(getattr(self, name) for name in _STATS)

    def rows(self) -> SimpleNamespace:
        """Zero-copy views of the live rows: the six leaves (differentiable views of the full leaves) and the three
        statistics.  For eager render_scene, filtering, PLY export and final_combine_all."""
        n = self.live_count
        return SimpleNamespace(**{name: getattr(self, name)[:n] for name in _FIELDS + _STATS})

    def param_groups(self, lrs: dict) -> list:
        """The reference's optimizer groups over the leaves: lrs maps xyz / f_dc / f_rest / opacity / scaling /
        rotation to a learning rate."""
        return [{"params": [getattr(self, _NAMES[k])], "lr": lr, "name": k} for k, lr in lrs.items()]

    # ---- events ------------------------------------------------------------------------------------------------
    def _live_params(self):
        n = self.live_count
        return {k: getattr(self, leaf).detach()[:n] for k, leaf in _NAMES.items()}

    def _moments(self, optimizer):
        """{densify name: (exp_avg, exp_avg_sq)} of the leaves that have Adam state (full tensors)."""
        out = {}
        if optimizer is None:
            return out
        for k, leaf in _NAMES.items():
            st = optimizer.state.get(getattr(self, leaf))
            if st:
                if st["exp_avg"].shape != getattr(self, leaf).shape or st["exp_avg_sq"].shape != getattr(self, leaf).shape:
                    raise ValueError(f"ReservedGroup: the Adam moments of {leaf} do not have the leaf's capacity")
                out[k] = (st["exp_avg"], st["exp_avg_sq"])
        return out

    def _commit(self, optimizer, new_p: dict, new_a: Optional[dict], n_out: int, stats=None):
        """Write an event's result rows [0, n_out) into the prefix (growing first if they do not fit)."""
        if n_out > self.capacity:
            self._grow(n_out, optimizer)
        with torch.no_grad():
            for k, t in new_p.items():
                getattr(self, _NAMES[k])[:n_out].copy_(t)
            moments = self._moments(optimizer)
            for k, (m1, m2) in (new_a or {}).items():
                if k in moments:
                    moments[k][0][:n_out].copy_(m1)
                    moments[k][1][:n_out].copy_(m2)
            for name in _STATS:
                t = getattr(self, name).view(-1)
                if stats is None:
                    t[:n_out].zero_()
                else:
                    t[:n_out].copy_(stats[name].reshape(-1))
            self.live.fill_(n_out)
        self.live_count = n_out

    def _grow(self, need: int, optimizer) -> None:
        """Re-allocate at capacity_for(need) with the live rows, moments and statistics copied, and move the optimizer's
        parameters and state to the new leaves (step counters kept)."""
        cap, n = capacity_for(need, self.headroom), self.live_count
        moments = self._moments(optimizer)
        with torch.no_grad():
            for k, leaf in _NAMES.items():
                old = getattr(self, leaf)
                new = torch.zeros((cap,) + tuple(old.shape[1:]), dtype=old.dtype, device=old.device)
                new[:n] = old[:n]
                new = torch.nn.Parameter(new.requires_grad_(old.requires_grad))
                setattr(self, leaf, new)
                if optimizer is None:
                    continue
                for group in optimizer.param_groups:
                    group["params"] = [new if p is old else p for p in group["params"]]
                st = optimizer.state.pop(old, None)
                if st is not None:
                    if k in moments:
                        for key in ("exp_avg", "exp_avg_sq"):
                            m = torch.zeros_like(new)
                            m[:n] = st[key][:n]
                            st[key] = m
                    optimizer.state[new] = st
            for name in _STATS:
                old = getattr(self, name)
                new = torch.zeros((cap,) + tuple(old.shape[1:]), dtype=old.dtype, device=old.device)
                new[:n] = old[:n]
                setattr(self, name, new)

    def densify_and_prune(self, optimizer, max_grad: float, min_opacity: float, extent: float, max_screen_size,
                          percent_dense: float = 0.01, N: int = 2, generator: Optional[torch.Generator] = None,
                          z: Optional[torch.Tensor] = None) -> dict:
        """The reference's densify_and_prune in place: densify.densify_and_prune over the live rows and their
        statistics (rows [kept | clones | split children], new moments zero, statistics zeroed), written back into the
        prefix.  -> densify's info."""
        n = self.live_count
        new_p, new_a, info = D.densify_and_prune(self._live_params(), {k: (m[:n], v[:n]) for k, (m, v) in
                                                                       self._moments(optimizer).items()} or None,
                                                 self.xyz_gradient_accum[:n], self.denom[:n], max_grad, min_opacity,
                                                 extent, max_screen_size, percent_dense, N, generator, z)
        self._commit(optimizer, new_p, new_a, int(info["points"]))
        return info

    def prune(self, mask: torch.Tensor, optimizer=None) -> None:
        """prune_points in place: drop the live rows where mask [live_count] is True from the leaves, the moments of
        `optimizer` (None: no Adam state yet) and the statistics (kept rows keep theirs)."""
        n = self.live_count
        if mask.numel() != n:
            raise ValueError(f"ReservedGroup.prune: mask has {mask.numel()} elements, the group has {n} live rows")
        stats = {name: getattr(self, name)[:n] for name in _STATS}
        new_p, new_a, new_s = D.prune_points(self._live_params(), {k: (m[:n], v[:n]) for k, (m, v) in
                                                                   self._moments(optimizer).items()} or None,
                                             stats, mask.reshape(-1))
        self._commit(optimizer, new_p, new_a, int(new_p["xyz"].shape[0]), stats=new_s)

    def filter(self, optimizer, settings_list, v_pow: float, prune_decay: float, prune_percent: float, *,
               views_per_pass: int = 16, score: Optional[torch.Tensor] = None) -> None:
        """The reference's gaussian_filtering in place: filtering.gaussian_filtering's score over rows(), then the
        prune of the rows at or below its percentile."""
        n = self.live_count
        stats = {name: getattr(self, name)[:n] for name in _STATS}
        new_p, new_a, new_s = F.gaussian_filtering(self._live_params(), {k: (m[:n], v[:n]) for k, (m, v) in
                                                                         self._moments(optimizer).items()} or None,
                                                   stats, settings_list, v_pow, prune_decay, prune_percent,
                                                   views_per_pass=views_per_pass, score=score)
        self._commit(optimizer, new_p, new_a, int(new_p["xyz"].shape[0]), stats=new_s)

    def reset_opacity(self, optimizer) -> None:
        """The reference's reset_opacity in place: opacity = inverse_sigmoid(min(sigmoid(opacity), 0.01)) on the live
        rows, whose opacity moments are zeroed (step counter kept)."""
        n = self.live_count
        with torch.no_grad():
            o = self._opacity[:n]
            new = torch.min(torch.sigmoid(o), torch.ones_like(o) * 0.01)
            o.copy_(torch.log(new / (1 - new)))
            st = optimizer.state.get(self._opacity) if optimizer is not None else None
            if st:
                st["exp_avg"][:n].zero_()
                st["exp_avg_sq"][:n].zero_()
