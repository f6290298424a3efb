"""The reference's Adam set-up and its in-place edits of the Adam state, restated for any torch.optim.Adam
subclass (harness code for the optimizer tests and benchmarks).

reference_adam builds the optimizer as training_setup does (/root/reference/gs_renderer.py:612-653: seven named
one-tensor groups, lr=0.0, eps=1e-15; learning rates of config.py:29-38).  The surgery functions follow
gs_renderer.py:854-930: the group named "background" is never edited, each function swaps in new nn.Parameters
and returns them by group name."""
import torch
from torch import nn

NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "background")
LRS = dict(xyz=0.00016, f_dc=0.005, f_rest=0.005 / 20, opacity=0.05, scaling=0.005, rotation=0.001,
           background=0.005)


def reference_adam(params, cls=torch.optim.Adam, **kwargs):
    """params: {group name: nn.Parameter} (any subset of NAMES, in that order)."""
    return cls([{"params": [params[k]], "lr": LRS[k], "name": k} for k in NAMES if k in params], lr=0.0, eps=1e-15,
               **kwargs)


def _swap(opt, group, new_param, edit_state):
    old = group["params"][0]
    state = opt.state.pop(old, None)
    group["params"][0] = new_param
    if state is not None:
        edit_state(state)
        opt.state[new_param] = state
    return new_param


def replace_tensor(opt, tensor, name):
    """replace_tensor_to_optimizer: the named parameter becomes `tensor`, its moments zeros, its step is kept."""
    out = {}
    for group in opt.param_groups:
        if group["name"] == name:
            def edit(st):
                st["exp_avg"] = torch.zeros_like(tensor)
                st["exp_avg_sq"] = torch.zeros_like(tensor)
            out[name] = _swap(opt, group, nn.Parameter(tensor.requires_grad_(True)), edit)
    return out


def prune(opt, keep):
    """_prune_optimizer: keep the rows where `keep` is True in every parameter and both moments."""
    out = {}
    for group in opt.param_groups:
        if group["name"] == "background":
            continue

        def edit(st):
            st["exp_avg"] = st["exp_avg"][keep]
            st["exp_avg_sq"] = st["exp_avg_sq"][keep]
        out[group["name"]] = _swap(opt, group, nn.Parameter(group["params"][0][keep].requires_grad_(True)), edit)
    return out


def cat_tensors(opt, tensors):
    """cat_tensors_to_optimizer: append rows to every parameter, with zero moments for them."""
    out = {}
    for group in opt.param_groups:
        if group["name"] == "background":
            continue
        ext = tensors[group["name"]]

        def edit(st):
            st["exp_avg"] = torch.cat((st["exp_avg"], torch.zeros_like(ext)), dim=0)
            st["exp_avg_sq"] = torch.cat((st["exp_avg_sq"], torch.zeros_like(ext)), dim=0)
        new = nn.Parameter(torch.cat((group["params"][0], ext), dim=0).requires_grad_(True))
        out[group["name"]] = _swap(opt, group, new, edit)
    return out
