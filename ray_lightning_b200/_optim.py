"""Which torch optimizers the fused steps take over, and what their kernels are given.

Both fused paths — the sharded step (K13, ``sharded.ShardedOptimizer``) and the step behind every DDP bucket (K14,
``comm.InBackwardOptimizer``) — compute torch's Adam / AdamW / SGD update themselves, so they may only take a
configuration whose update they implement.  That decision is an allow-list over the options of the optimizer
(the keys of its ``defaults``): every option is either read here and handed to the kernel, or known to change only
how torch rounds (``_ROUNDING_ONLY``), or has to sit at the value torch's own constructor defaults it to.  An option
torch adds later is therefore at worst a reason not to fuse, never a silently ignored change of arithmetic.  Group
keys outside ``defaults`` (``initial_lr`` and OneCycleLR's ``max_lr``, ``min_lr``, ... that lr schedulers add) are
not options and are ignored."""
import functools
import inspect

import torch

# the options each class's kernels implement, read per parameter group by kernel_args()
_HANDLED = {
    torch.optim.Adam: ("lr", "betas", "eps", "weight_decay", "decoupled_weight_decay"),
    torch.optim.AdamW: ("lr", "betas", "eps", "weight_decay", "decoupled_weight_decay"),
    torch.optim.SGD: ("lr", "momentum", "weight_decay"),
}
# torch's choice of implementation: the same update, rounded differently (the fused kernels round like the default
# foreach path; DESIGN §3 gives the contract for the others)
_ROUNDING_ONLY = ("foreach", "fused", "differentiable")


class NotFusable(ValueError):
    """A configuration the fused kernels do not implement; the message names the option."""


@functools.lru_cache(maxsize=None)      # kernel_args runs at every step: look the signature up once
def _signature_default(cls, key):
    p = inspect.signature(cls.__init__).parameters.get(key)
    return inspect.Parameter.empty if p is None else p.default


def _is(value, default):
    return not isinstance(value, torch.Tensor) and value is not inspect.Parameter.empty and value == default


def kernel_args(cls, defaults, group):
    """The fused kernels' arguments for one parameter group of a ``cls`` optimizer whose options are the keys of
    ``defaults``: ``lr``, ``beta1``, ``beta2``, ``eps``, ``weight_decay`` and ``adamw`` (decoupled decay) for Adam and
    AdamW; ``lr``, ``momentum`` and ``weight_decay`` for SGD.  Raises NotFusable naming the option otherwise."""
    handled = _HANDLED.get(cls)
    if handled is None:
        raise NotFusable("the fused step implements torch.optim.Adam, AdamW and SGD (got %s)" % cls.__name__)
    for key in defaults:
        if key in handled or key in _ROUNDING_ONLY:
            continue
        default = _signature_default(cls, key)
        if not _is(group.get(key, default), default):
            raise NotFusable("the fused %s step does not implement %s=%r" % (cls.__name__, key, group.get(key)))
    if isinstance(group["lr"], torch.Tensor) and cls is not torch.optim.SGD:
        raise NotFusable("the fused %s step takes a float lr, not a tensor" % cls.__name__)
    if cls is torch.optim.SGD:
        return dict(lr=float(group["lr"]), momentum=float(group.get("momentum", 0.0)),
                    weight_decay=float(group.get("weight_decay", 0.0)))
    # torch's Adam.step reads the flag per group; AdamW is Adam with it set (and a group may clear it)
    decoupled = group.get("decoupled_weight_decay", cls is torch.optim.AdamW)
    return dict(lr=float(group["lr"]), beta1=float(group["betas"][0]), beta2=float(group["betas"][1]),
                eps=float(group["eps"]), weight_decay=float(group["weight_decay"]), adamw=int(bool(decoupled)))
