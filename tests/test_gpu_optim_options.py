"""Every fused Adam / AdamW / SGD configuration of both optimizer paths on an H100, one step from captured state, bit
for bit against torch's CUDA optimizer of the same options in its default (foreach) form.

Two worker processes share the device over a gloo control plane.  Each step is compared from the state captured just
before it (the owner's reduced gradient, or DDP's averaged ``p.grad``), so the result does not depend on how the
gradients were summed.  Options that change only torch's rounding (``foreach=False``, ``fused=True``) are held to the
float64 bound of tests/optim_ref.py instead, as is torch's own result for them."""
import os
import socket
from contextlib import closing

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import optim_ref as ref
from test_gpu_optim import assert_same_bits, bound_excess

pytestmark = pytest.mark.gpu

Adam, AdamW, SGD = torch.optim.Adam, torch.optim.AdamW, torch.optim.SGD
ROUNDING_ONLY = ("foreach", "fused", "differentiable")
T = torch.tensor

# name -> (class, constructor options, per-group overrides of the two-group split or None)
ADAM_CASES = {
    "adam": (Adam, dict(lr=1e-2, weight_decay=0.0), None),
    "adam_l2": (Adam, dict(lr=1e-2, weight_decay=0.1), None),
    "adam_decoupled": (Adam, dict(lr=1e-2, weight_decay=0.1, decoupled_weight_decay=True), None),
    "adamw": (AdamW, dict(lr=1e-2, weight_decay=0.05), None),
    "adamw_coupled_group": (AdamW, dict(lr=1e-2, weight_decay=0.05), [dict(decoupled_weight_decay=False)]),
    "adam_tensor_betas": (Adam, dict(lr=1e-2, betas=(T(0.8), T(0.99)), weight_decay=0.1), None),
    "adam_single_tensor": (Adam, dict(lr=1e-2, weight_decay=0.1, foreach=False), None),
    "adamw_fused": (AdamW, dict(lr=1e-2, weight_decay=0.05, fused=True), None),
}
SHARDED_CASES = dict(ADAM_CASES, adam_two_groups=(
    Adam, dict(lr=1e-2, weight_decay=0.1), [dict(decoupled_weight_decay=True), dict(decoupled_weight_decay=False, lr=3e-3)]))
SGD_CASES = {
    "sgd": (SGD, dict(lr=0.05), None),
    "sgd_wd": (SGD, dict(lr=0.05, weight_decay=1e-2), None),
    "sgd_tensor_wd": (SGD, dict(lr=0.05, weight_decay=T(1e-2)), None),
    "sgd_momentum": (SGD, dict(lr=0.05, momentum=0.9), None),
    "sgd_momentum_wd": (SGD, dict(lr=0.05, momentum=0.9, weight_decay=1e-2), None),
    "sgd_momentum_tensor_wd": (SGD, dict(lr=0.05, momentum=0.9, weight_decay=T(1e-2)), None),
    "sgd_single_tensor": (SGD, dict(lr=0.05, momentum=0.9, weight_decay=1e-2, foreach=False), None),
    "sgd_fused": (SGD, dict(lr=0.05, momentum=0.9, weight_decay=1e-2, fused=True), None),
}
IN_BACKWARD_CASES = dict({k: v for k, v in ADAM_CASES.items()}, **SGD_CASES)


def _port():
    with closing(socket.socket(socket.AF_INET, socket.SOCK_STREAM)) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _net(dev):
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(24, 300), torch.nn.Tanh(), torch.nn.Linear(300, 40), torch.nn.Tanh(),
                               torch.nn.Linear(40, 5)).to(dev)


def _groups(model, overrides):
    if overrides is None:
        return [{"params": list(model.parameters())}]
    if len(overrides) == 1:
        return [dict(overrides[0], params=list(model.parameters()))]
    biases = [p for n, p in model.named_parameters() if not n.endswith("weight")]
    weights = [p for n, p in model.named_parameters() if n.endswith("weight")]
    return [dict(overrides[0], params=biases), dict(overrides[1], params=weights)]


def _options(group):
    return {k: v for k, v in group.items() if k != "params"}


def _foreach_form(opts):
    """The same update in torch's default CUDA form: rounding-only options dropped, tensor options as the doubles they
    hold (torch's foreach Adam refuses tensor betas)."""
    as_double = lambda v: (tuple(as_double(x) for x in v) if isinstance(v, tuple)
                           else float(v) if isinstance(v, torch.Tensor) else v)
    return {k: as_double(v) for k, v in opts.items() if k not in ROUNDING_ONLY}


def _hp(cls, opts):
    """The update's hyper-parameters as optim_ref takes them."""
    f = _foreach_form(opts)
    if cls is SGD:
        return dict(lr=f["lr"], momentum=f.get("momentum", 0.0), weight_decay=f.get("weight_decay", 0.0))
    return dict(lr=f["lr"], beta1=f["betas"][0], beta2=f["betas"][1], eps=f["eps"], weight_decay=f["weight_decay"],
                adamw=bool(f.get("decoupled_weight_decay", cls is AdamW)))


def _rounding_only(opts):
    return opts.get("foreach") is False or bool(opts.get("fused"))


def _torch_step(cls, opts, p, g, state):
    """One step of ``cls`` with group options ``opts`` on clones; returns (parameter, state after)."""
    prm = torch.nn.Parameter(p.clone())
    opt = cls([dict(opts, params=[prm])])
    if state:      # torch's fused kernels keep the step count on the device
        opt.state[prm] = {k: v.to(p.device) if k == "step" and opts.get("fused") else v.clone() for k, v in state.items()}
    prm.grad = g.clone()
    opt.step()
    return prm.detach(), opt.state[prm]


def _np(t):
    return t.detach().float().cpu().numpy().reshape(-1)


def _adam_bound(p, g, m, v, hp, step, got):
    out64, tol = ref.adam_step64(p, g, m, v, step=step, **hp)
    ok = np.isfinite(g)
    for x in out64:
        ok &= np.isfinite(x)
    return bound_excess(got, out64, tol, ok)


def _sgd_bound(p, g, buf, hp, got_p):
    out64, _ = ref.sgd_step64(p, g, buf, **hp)
    tol_p, _ = ref.sgd_bound64(p, g, buf, **hp)
    return bound_excess([got_p], [out64], [tol_p], np.isfinite(out64))


def _setup(rank, world, port):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, init_method="env://")
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    return dist, dev


def _batch(rank, it, dev):
    g = torch.Generator().manual_seed(100 * it + rank)
    return torch.randn(16, 24, generator=g).to(dev), torch.randn(16, 5, generator=g).to(dev)


# ---- the sharded step ------------------------------------------------------------------------------------------------------
def _sharded_worker(rank, world, port, ret):
    from ray_lightning_b200.comm import Communicator
    from ray_lightning_b200.sharded import FlatShards, ShardedOptimizer, group_index_of
    dist, dev = _setup(rank, world, port)
    errors, excess = [], {}
    try:
        for name, (cls, kw, overrides) in SHARDED_CASES.items():
            model = _net(dev)
            base = cls(_groups(model, overrides), **kw)
            comm = Communicator(rank, world, dev.index, 64 << 20, mem="ipc", timeout_ms=60000)
            shards = FlatShards(model, comm, wire="fp32", group_of=group_index_of(list(model.parameters()), base),
                                reduce_bucket_mb=0.02)
            sopt = ShardedOptimizer(base, shards, wire="fp32", stream=torch.cuda.Stream(priority=-1))
            if not sopt.fused:
                errors.append("%s: not fused" % name)
            for it in (0, 1):
                sopt.zero_grad()
                x, y = _batch(rank, it, dev)
                torch.nn.functional.mse_loss(model(x), y).backward()
                if it == 0:
                    sopt.step()
            # the state is read only after every rank's backward and exchanges have finished
            torch.cuda.synchronize()
            dist.barrier()
            n_own = shards.own.stop - shards.own.start
            red = shards.reduced[:n_own].clone()
            p0 = shards.flat_params[shards.own].clone()
            m0, v0 = sopt.exp_avg[:n_own].clone(), sopt.exp_avg_sq[:n_own].clone()
            sopt.step()
            torch.cuda.synchronize()
            got = (shards.flat_params[shards.own], sopt.exp_avg[:n_own], sopt.exp_avg_sq[:n_own])
            for gi, (lo, hi) in enumerate(sopt.group_range):
                if hi == lo:
                    continue
                opts = _options(sopt.param_groups[gi])
                state = {"step": T(1.0), "exp_avg": m0[lo:hi], "exp_avg_sq": v0[lo:hi]}
                wp, ws = _torch_step(cls, _foreach_form(opts), p0[lo:hi], red[lo:hi], state)
                what = "%s group %d rank %d" % (name, gi, rank)
                mine = [_np(t[lo:hi]) for t in got]
                for k, a, b in zip("pmv", mine, (wp, ws["exp_avg"], ws["exp_avg_sq"])):
                    try:
                        assert_same_bits(a, _np(b), "%s %s" % (what, k))
                    except AssertionError as e:
                        errors.append(str(e))
                if not torch.equal(red, shards.reduced[:n_own]):
                    errors.append("%s: the reduced gradient changed during step()" % what)
                if _rounding_only(opts):
                    args = [_np(t) for t in (p0[lo:hi], red[lo:hi], m0[lo:hi], v0[lo:hi])]
                    hp = _hp(cls, opts)
                    tp, ts = _torch_step(cls, opts, p0[lo:hi], red[lo:hi], state)
                    excess[(name, gi)] = {"ours": _adam_bound(*args, hp, 2, mine),
                                          "torch": _adam_bound(*args, hp, 2, [_np(tp), _np(ts["exp_avg"]),
                                                                              _np(ts["exp_avg_sq"])])}
            for p in shards.params:          # parameters were views of the arena: ordinary storage before it goes
                p.data = p.data.clone()
                p.grad = None
            del sopt, shards
            comm.close()
        ret[rank] = {"errors": errors, "excess": excess}
    finally:
        dist.destroy_process_group()


# ---- the step behind every DDP bucket ------------------------------------------------------------------------------------
def _in_backward_worker(rank, world, port, ret):
    from torch.nn.parallel import DistributedDataParallel as DDP
    from ray_lightning_b200.comm import B200HookState, InBackwardOptimizer, b200_allreduce_hook
    dist, dev = _setup(rank, world, port)
    errors, excess, states = [], {}, []
    try:
        for name, (cls, kw, overrides) in IN_BACKWARD_CASES.items():
            model = _net(dev)
            ddp = DDP(model, device_ids=[dev.index], bucket_cap_mb=0.25, gradient_as_bucket_view=True)
            st = B200HookState(wire="fp32", total_grad_elems=sum(p.numel() for p in model.parameters()), mem="ipc")
            states.append(st)
            ddp.register_comm_hook(st, b200_allreduce_hook)
            opt = InBackwardOptimizer(cls(_groups(ddp, overrides), **kw), st)
            params = opt.param_groups[0]["params"]
            for step in (1, 2):
                before = [p.detach().clone() for p in params]
                sd = opt.state_dict()
                opt.zero_grad(set_to_none=False)
                x, y = _batch(rank, step, dev)
                torch.nn.functional.mse_loss(ddp(x), y).backward()
                torch.cuda.synchronize()
                dist.barrier()
                opts = _options(opt.param_groups[0])
                hp = _hp(cls, opts)
                for i, (p, p0) in enumerate(zip(params, before)):
                    state = sd["state"].get(i, {})
                    wp, _ = _torch_step(cls, _foreach_form(opts), p0, p.grad, state)
                    what = "%s step %d param %d rank %d" % (name, step, i, rank)
                    try:
                        assert_same_bits(_np(p), _np(wp), what)
                    except AssertionError as e:
                        errors.append(str(e))
                    if _rounding_only(opts):
                        tp, ts = _torch_step(cls, opts, p0, p.grad, state)
                        g = _np(p.grad)
                        if cls is SGD:
                            buf = _np(state["momentum_buffer"]) if "momentum_buffer" in state else None
                            res = {"ours": _sgd_bound(_np(p0), g, buf, hp, _np(p)),
                                   "torch": _sgd_bound(_np(p0), g, buf, hp, _np(tp))}
                        else:
                            m = _np(state["exp_avg"]) if state else np.zeros_like(g)
                            v = _np(state["exp_avg_sq"]) if state else np.zeros_like(g)
                            s = opt._pstate[id(p)]
                            res = {"ours": _adam_bound(_np(p0), g, m, v, hp, step, [_np(p), _np(s[0]), _np(s[1])]),
                                   "torch": _adam_bound(_np(p0), g, m, v, hp, step,
                                                        [_np(tp), _np(ts["exp_avg"]), _np(ts["exp_avg_sq"])])}
                        excess[(name, step, i)] = res
                opt.step()
            if opt.applied < 2:
                errors.append("%s: K14 ran %d times" % (name, opt.applied))
        ret[rank] = {"errors": errors, "excess": excess}
    finally:
        for st in states:
            st.close()
        dist.destroy_process_group()


def _report(ret):
    """Every rank's mismatches, and the bound checks: ours always, torch's single-tensor path too (DESIGN §3); torch's
    fused kernels are measured and printed."""
    errors = []
    for r in sorted(ret.keys()):
        errors += ret[r]["errors"]
        for key, res in sorted(ret[r]["excess"].items(), key=str):
            for who in ("ours", "torch"):
                bad = [(k, n, round(worst, 3)) for k, (n, worst) in zip("pmv", res[who]) if n]
                fused = "fused" in key[0]
                print("bound %s rank %d %s: %s" % (who, r, key, bad or "inside (worst %.3f)" % max(w for _, w in res[who])))
                if bad and (who == "ours" or not fused):
                    errors.append("%s rank %d %s outside the float64 bound: %s" % (who, r, key, bad))
    assert not errors, "\n".join(errors[:20])


def test_sharded_step_matches_torch_for_every_fused_configuration():
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_sharded_worker, args=(2, _port(), ret), nprocs=2, join=True)
    assert sorted(ret.keys()) == [0, 1]
    assert len(ret[0]["excess"]) + len(ret[1]["excess"]) >= 4         # foreach=False and fused=True, on both ranks
    _report(ret)


def test_in_backward_step_matches_torch_for_every_configuration():
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_in_backward_worker, args=(2, _port(), ret), nprocs=2, join=True)
    assert sorted(ret.keys()) == [0, 1]
    _report(ret)
