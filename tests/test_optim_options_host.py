"""Every option of torch's Adam, AdamW and SGD through both fused optimizer paths, on CPU.

The sharded step (K13 behind ``ShardedOptimizer``) and the step behind every DDP bucket (K14 behind
``InBackwardOptimizer``) compute torch's update themselves.  ``ray_lightning_b200._optim.kernel_args`` decides
which configurations they take and what reaches the kernels; OPTIONS below states, for every key of each class's
``defaults``, the values tried and the outcome expected on each path.  The sharded path runs on the threaded
communicator double of test_sharded_host.py (its adam_push_ steps torch's optimizer with the kernel arguments it is
handed); the in-backward path records what it would launch, and the recorded arguments are stepped with the fp32
restatement of tests/optim_ref.py against torch's own update in float64."""
import inspect

import numpy as np
import pytest
import torch

import optim_ref as ref
from ray_lightning_b200.comm import B200HookState, InBackwardOptimizer
from ray_lightning_b200.sharded import FlatShards, ShardedOptimizer, group_index_of
from test_comm_host import _FakeComm
from test_sharded_host import FakeComm, _Net, make_model, run_ranks

Adam, AdamW, SGD = torch.optim.Adam, torch.optim.AdamW, torch.optim.SGD
F, G, R = "fused", "generic", "refused"
f32 = np.float32

# the configuration every row starts from, and the kernel arguments it gives
BASE = {Adam: dict(lr=1e-2, betas=(0.8, 0.99), eps=1e-7, weight_decay=0.1),
        AdamW: dict(lr=1e-2, betas=(0.8, 0.99), eps=1e-7, weight_decay=0.1),
        SGD: dict(lr=0.05, momentum=0.9, weight_decay=0.01)}
BASE_ARGS = {Adam: dict(lr=1e-2, beta1=0.8, beta2=0.99, eps=1e-7, weight_decay=0.1, adamw=0),
             AdamW: dict(lr=1e-2, beta1=0.8, beta2=0.99, eps=1e-7, weight_decay=0.1, adamw=1),
             SGD: dict(lr=0.05, momentum=0.9, weight_decay=0.01)}
T = torch.tensor


def _f(x):
    """The double a 1-element fp32 tensor option stands for."""
    return float(T(x))


def _adam_rows(decoupled_default):
    return {
        "lr": [(3e-3, F, F, dict(lr=3e-3)), (T(3e-3), G, R, None)],
        "betas": [((0.5, 0.9), F, F, dict(beta1=0.5, beta2=0.9)),
                  ((0.0, 0.999), F, F, dict(beta1=0.0, beta2=0.999)),
                  ((T(0.5), T(0.9)), F, F, dict(beta1=_f(0.5), beta2=_f(0.9)))],
        "eps": [(1e-6, F, F, dict(eps=1e-6))],
        "weight_decay": [(0.0, F, F, dict(weight_decay=0.0)), (0.3, F, F, dict(weight_decay=0.3))],
        "decoupled_weight_decay": [(not decoupled_default, F, F, dict(adamw=int(not decoupled_default))),
                                   (decoupled_default, F, F, {})],
        "amsgrad": [(True, G, R, None), (False, F, F, {})],
        "maximize": [(True, G, R, None), (False, F, F, {})],
        "capturable": [(True, G, R, None), (False, F, F, {})],
        "foreach": [(True, F, F, {}), (False, F, F, {})],
        "fused": [(True, F, F, {}), (False, F, F, {})],
        "differentiable": [(True, F, F, {})],
    }


# class -> option -> [(value, sharded outcome, in-backward outcome, kernel arguments that differ from BASE_ARGS)]
OPTIONS = {
    Adam: _adam_rows(False),
    AdamW: _adam_rows(True),
    SGD: {    # the sharded path has no fused SGD: every SGD configuration runs torch's step on the owned shard
        "lr": [(0.01, G, F, dict(lr=0.01)), (T(0.01), G, F, dict(lr=_f(0.01)))],
        "momentum": [(0.0, G, F, dict(momentum=0.0)), (0.5, G, F, dict(momentum=0.5))],
        "dampening": [(0.1, G, R, None), (0.0, G, F, {})],
        "weight_decay": [(0.0, G, F, dict(weight_decay=0.0)), (T(1e-2), G, F, dict(weight_decay=_f(1e-2)))],
        "nesterov": [(True, G, R, None), (False, G, F, {})],
        "maximize": [(True, G, R, None)],
        "foreach": [(True, G, F, {}), (False, G, F, {})],
        "fused": [(True, G, F, {})],
        "differentiable": [(True, G, F, {})],
    },
}
ROUNDING_ONLY = ("foreach", "fused", "differentiable")
# torch itself cannot step these on CPU (capturable wants device tensors): only the path decision is checked
CPU_UNSTEPPABLE = {"capturable": True}

ROWS = [pytest.param(cls, key, i, id="%s-%s-%d" % (cls.__name__, key, i))
        for cls, opts in OPTIONS.items() for key, vals in opts.items() for i in range(len(vals))]


def make(cls, params, key=None, value=None):
    """A ``cls`` optimizer in the BASE configuration with ``key`` set to ``value``: through the constructor when it
    takes the option, otherwise (AdamW's decoupled_weight_decay) in the parameter group."""
    kw, group = dict(BASE[cls]), {"params": list(params)}
    if key in inspect.signature(cls.__init__).parameters:
        kw[key] = value
    elif key is not None:
        group[key] = value
    return cls([group], **kw)


def make_ref(cls, params, key, value):
    """The plain torch optimizer the row must match: the same update, rounding-only options left at their default."""
    return make(cls, params) if key in ROUNDING_ONLY else make(cls, params, key, value)


def _data(world, steps):
    return [[(torch.randn(6, 13, generator=torch.Generator().manual_seed(100 * s + r)),
              torch.randn(6, 3, generator=torch.Generator().manual_seed(7 + 100 * s + r))) for r in range(world)]
            for s in range(steps)]


class RecordingComm(FakeComm):
    """The communicator double, keeping the Adam groups every fused step hands to the push."""

    def adam_push_(self, params, exp_avg, exp_avg_sq, reduced, shard_off, groups, **kw):
        self.__dict__.setdefault("pushed", []).append([dict(a) for _, _, a in groups])
        return super().adam_push_(params, exp_avg, exp_avg_sq, reduced, shard_off, groups, **kw)


KERNEL_KEYS = ("lr", "beta1", "beta2", "eps", "weight_decay", "adamw")


def run_sharded(world, build, build_ref, steps=5, sched=None):
    """W ranks step ``build(model)`` through ShardedOptimizer; one replica steps ``build_ref(model)`` on the mean
    gradient.  Returns per rank (parameters, sopt.fused, groups pushed per step, final param_groups), and the
    reference parameters."""
    net = _Net(world)
    data = _data(world, steps)
    models = [make_model() for _ in range(world)]

    def rank_fn(r):
        model = models[r]
        comm = RecordingComm(net, r)
        base = build(model)
        params = [p for p in model.parameters()]
        shards = FlatShards(model, comm, wire="fp32", group_of=group_index_of(params, base), reduce_bucket_mb=0.001)
        sopt = ShardedOptimizer(base, shards, wire="fp32")
        s = sched(sopt) if sched else None
        for k in range(steps):
            sopt.zero_grad()
            x, y = data[k][r]
            torch.nn.functional.mse_loss(model(x), y).backward()
            sopt.step()
            if s is not None:
                s.step()
        return ([p.detach().clone() for p in params], sopt.fused, comm.__dict__.get("pushed", []),
                [{k: v for k, v in g.items() if k != "params"} for g in sopt.param_groups])

    outs = run_ranks(world, rank_fn)
    refm = make_model()
    ref_opt = build_ref(refm)
    s = sched(ref_opt) if sched else None
    for k in range(steps):
        ref_opt.zero_grad()
        for r in range(world):
            x, y = data[k][r]
            (torch.nn.functional.mse_loss(refm(x), y) / world).backward()
        ref_opt.step()
        if s is not None:
            s.step()
    return outs, [p.detach() for p in refm.parameters()]


def _assert_matches(outs, want):
    for params, *_ in outs:
        for a, b in zip(params, want):
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def _kernel_view(a):
    return {k: a[k] for k in KERNEL_KEYS}


# ---- the table covers every option ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("cls", list(OPTIONS), ids=lambda c: c.__name__)
def test_table_covers_every_option(cls):
    """A torch release that adds an option fails here by name until the table (and kernel_args) say what it means."""
    defaults = cls([torch.nn.Parameter(torch.zeros(1))]).defaults
    missing = sorted(set(defaults) - set(OPTIONS[cls]))
    assert not missing, "%s options without a row: %s" % (cls.__name__, missing)
    stale = sorted(set(OPTIONS[cls]) - set(defaults))
    assert not stale, "%s rows for options torch does not have: %s" % (cls.__name__, stale)
    kw = [k for k in inspect.signature(cls.__init__).parameters if k not in ("self", "params")]
    assert not set(kw) - set(defaults), "%s constructor keywords outside defaults: %s" % (cls.__name__, set(kw) - set(defaults))


# ---- the sharded path --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("cls,key,i", ROWS)
def test_sharded_option(cls, key, i, world):
    value, outcome, _, args = OPTIONS[cls][key][i]
    if CPU_UNSTEPPABLE.get(key) == value:
        model = make_model()
        base = make(cls, model.parameters(), key, value)
        shards = FlatShards(model, RecordingComm(_Net(1), 0), wire="fp32")
        sopt = ShardedOptimizer(base, shards, wire="fp32")
        assert sopt.fused == (outcome == F)
        return
    outs, want = run_sharded(world, lambda m: make(cls, m.parameters(), key, value),
                             lambda m: make_ref(cls, m.parameters(), key, value))
    for params, fused, pushed, _ in outs:
        assert fused == (outcome == F), (key, value)
        if fused:
            assert len(pushed) == 5
            for k, groups in enumerate(pushed):
                for a in groups:
                    assert _kernel_view(a) == dict(BASE_ARGS[cls], **args) and a["step"] == k + 1
        else:
            assert all(groups == [] for groups in pushed)
    _assert_matches(outs, want)


def _two_groups(model, first, second):
    weights = [p for n, p in model.named_parameters() if n.endswith("weight")]
    biases = [p for n, p in model.named_parameters() if not n.endswith("weight")]
    return [dict(first, params=biases), dict(second, params=weights)]


# (class, options of the bias group, options of the weight group, kernel arguments of each, fused)
TWO_GROUPS = [
    (Adam, dict(decoupled_weight_decay=True, lr=2e-2), dict(weight_decay=0.05),
     [dict(adamw=1, lr=2e-2), dict(weight_decay=0.05)], True),
    (AdamW, dict(decoupled_weight_decay=False, betas=(0.5, 0.95)), dict(eps=1e-5),
     [dict(adamw=0, beta1=0.5, beta2=0.95), dict(eps=1e-5)], True),
    (AdamW, dict(weight_decay=0.0), dict(amsgrad=True), None, False),
    (Adam, dict(foreach=False), dict(fused=True, decoupled_weight_decay=True), [{}, dict(adamw=1)], True),
]


@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("case", range(len(TWO_GROUPS)))
def test_sharded_per_group_options(case, world):
    """Options set per parameter group: each group's own decoupled flag and constants reach its slice of the shard;
    one group with an option K13 lacks sends the whole optimizer to the generic step."""
    cls, first, second, args, fused = TWO_GROUPS[case]
    strip = lambda d: {k: v for k, v in d.items() if k not in ROUNDING_ONLY}
    outs, want = run_sharded(world, lambda m: cls(_two_groups(m, first, second), **BASE[cls]),
                             lambda m: cls(_two_groups(m, strip(first), strip(second)), **BASE[cls]))
    for params, is_fused, pushed, groups in outs:
        assert is_fused == fused
        assert [g.get("decoupled_weight_decay") for g in groups] == [
            d.get("decoupled_weight_decay", cls is AdamW) for d in (first, second)]
        if fused:
            seen = {}
            for step_groups in pushed:
                for a in step_groups:
                    seen.setdefault(a["adamw"], _kernel_view(a))
            want_args = [dict(BASE_ARGS[cls], **a) for a in args]
            for got in seen.values():        # a rank pushes only the groups it owns a part of
                assert got in want_args
    _assert_matches(outs, want)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_one_cycle_scheduler_keeps_adam_fused(world):
    """OneCycleLR adds initial_lr, max_lr, min_lr, base_momentum and max_momentum to every group and cycles lr and
    beta1: keys outside the optimizer's options, so the step stays fused and follows the schedule."""
    sched = lambda o: torch.optim.lr_scheduler.OneCycleLR(o, max_lr=5e-2, total_steps=10)
    outs, want = run_sharded(world, lambda m: make(Adam, m.parameters(), "decoupled_weight_decay", True),
                             lambda m: make(Adam, m.parameters(), "decoupled_weight_decay", True), sched=sched)
    for params, fused, pushed, groups in outs:
        assert fused and {"initial_lr", "max_lr", "min_lr", "base_momentum", "max_momentum"} <= set(groups[0])
        lrs = [step_groups[0]["lr"] for step_groups in pushed if step_groups]
        beta1s = [step_groups[0]["beta1"] for step_groups in pushed if step_groups]
        assert lrs and len(set(lrs)) == len(lrs) and len(set(beta1s)) > 1
        assert all(a["adamw"] == 1 for step_groups in pushed for a in step_groups)
    _assert_matches(outs, want)


# ---- the in-backward path ----------------------------------------------------------------------------------------------
class _GradBucket:
    """CPU stand-in for dist.GradBucket: the parameters, their gradients as views of one flat buffer."""

    def __init__(self, params, flat):
        self._params, self._flat = params, flat
        self._grads, off = [], 0
        for p in params:
            self._grads.append(flat[off:off + p.numel()].view(p.shape))
            off += p.numel()

    def parameters(self):
        return self._params

    def gradients(self):
        return self._grads

    def index(self):
        return 0


SHAPES = [(37,), (5, 3), (1,)]


def _float64_semantics(cls, key, value, params64, state64):
    """torch's own update of the row's configuration in float64; tensor options enter as the doubles they hold."""
    as_double = (lambda v: tuple(as_double(x) for x in v) if isinstance(v, tuple)
                 else float(v) if isinstance(v, torch.Tensor) else v)
    opt = make(cls, params64) if key in ROUNDING_ONLY else make(cls, params64, key, as_double(value))
    for p, st in zip(params64, state64):
        if st:
            opt.state[p] = st
    opt.step()
    return opt


@pytest.mark.parametrize("cls,key,i", ROWS)
def test_in_backward_option(cls, key, i):
    value, _, outcome, args = OPTIONS[cls][key][i]
    params = [torch.nn.Parameter(torch.from_numpy(ref.state(int(np.prod(s)), 3 + k)[0]).view(s)) for k, s in enumerate(SHAPES)]
    base = make(cls, params, key, value)
    if outcome == R:
        with pytest.raises(ValueError, match=key):
            InBackwardOptimizer(base, B200HookState(wire="fp32", total_grad_elems=1))
        return
    opt = InBackwardOptimizer(base, B200HookState(wire="fp32", total_grad_elems=1))
    comm = _FakeComm()
    n = sum(p.numel() for p in params)
    want_args = dict(BASE_ARGS[cls], **args)
    adam = cls is not SGD
    for step in (1, 2):
        g = ref.grads(n, 50 + step, edges=False)
        flat = torch.from_numpy(g.copy())
        p0 = np.concatenate([p.detach().reshape(-1).numpy() for p in params])
        # the state K14 would step from: zeros before step 1 (torch starts there too), random before step 2
        if step == 2:
            _, m0, v0 = ref.state(n, 9)
            off = 0
            for p in params:
                s1, s2 = opt._states(p)
                if s1 is not None:
                    s1.view(-1).copy_(torch.from_numpy(m0[off:off + p.numel()]))
                if s2 is not None:
                    s2.view(-1).copy_(torch.from_numpy(np.abs(v0[off:off + p.numel()])))
                off += p.numel()
        st1 = [opt._states(p)[0] for p in params]
        st2 = [opt._states(p)[1] for p in params]
        m = None if st1[0] is None else np.concatenate([s.reshape(-1).numpy() for s in st1])
        v = None if st2[0] is None else np.concatenate([s.reshape(-1).numpy() for s in st2])
        opt.apply_bucket(comm, _GradBucket(params, flat), flat, None)
        idx, ptr, numel, kind, hp, mom, _ = comm.ctx.applied[-1]
        assert (idx, ptr, numel, kind) == (0, flat.data_ptr(), n, int(adam))
        got = dict(lr=hp.lr, weight_decay=hp.weight_decay)
        if adam:
            got.update(beta1=hp.beta1, beta2=hp.beta2, eps=hp.eps, adamw=hp.adamw)
        else:
            got.update(momentum=f32(mom))
            want_args = dict(want_args, momentum=f32(want_args["momentum"]))
        assert got == want_args and hp.step == step and hp.zero_grads == 0
        # what K14 computes from the recorded arguments, against torch's update of this configuration in float64
        p64 = [torch.nn.Parameter(p.detach().double().clone()) for p in params]
        off, state64 = 0, []
        for p, q in zip(params, p64):
            k = p.numel()
            q.grad = torch.from_numpy(g[off:off + k].astype(np.float64)).view(p.shape)
            if adam:
                state64.append({"step": T(float(step - 1)), "exp_avg": torch.from_numpy(m[off:off + k].astype(np.float64)).view(p.shape),
                                "exp_avg_sq": torch.from_numpy(v[off:off + k].astype(np.float64)).view(p.shape)} if step > 1 else {})
            else:
                state64.append({"momentum_buffer": torch.from_numpy(m[off:off + k].astype(np.float64)).view(p.shape)}
                               if step > 1 and m is not None else {})
            off += k
        _float64_semantics(cls, key, value, p64, state64)
        want64 = np.concatenate([q.detach().reshape(-1).numpy() for q in p64])
        if adam:
            hp32 = dict(lr=hp.lr, beta1=hp.beta1, beta2=hp.beta2, eps=hp.eps, weight_decay=hp.weight_decay,
                        adamw=bool(hp.adamw))
            got32 = ref.adam_step32(p0, g, m, v, step=hp.step, **hp32)[0]
            tol = ref.adam_step64(p0, g, m, v, step=step, **dict(want_args, adamw=bool(want_args["adamw"])))[1][0]
        else:
            buf = m if (step > 1 and m is not None) else None
            sgd = dict(lr=hp.lr, momentum=float(mom), weight_decay=hp.weight_decay)
            got32 = ref.sgd_step32(p0, g, buf, **sgd)[0]
            tol = ref.sgd_bound64(p0, g, buf, lr=want_args["lr"], momentum=float(want_args["momentum"]),
                                  weight_decay=want_args["weight_decay"])[0]
        err = np.abs(got32.astype(np.float64) - want64)
        bad = ~(err <= tol + np.spacing(np.abs(got32)).astype(np.float64) / 2)
        assert not bad.any(), "%s=%r step %d: %d of %d outside the float64 bound, worst %g" % (
            key, value, step, bad.sum(), n, (err / tol).max())
        opt.step()


# ---- checkpoints keep the flag per group -----------------------------------------------------------------------------------
def test_decoupled_flag_survives_checkpoints():
    """consolidated_state_dict / state_dict carry decoupled_weight_decay per group; torch's own Adam loads the result,
    and both wrappers built from a plain Adam step with the loaded flags."""
    first, second = dict(decoupled_weight_decay=True), dict(decoupled_weight_decay=False)
    net = _Net(2)
    models = [make_model() for _ in range(2)]
    data = _data(2, 2)

    def rank_fn(r):
        model = models[r]
        base = Adam(_two_groups(model, first, second), **BASE[Adam])
        shards = FlatShards(model, FakeComm(net, r), wire="fp32", group_of=group_index_of(list(model.parameters()), base))
        sopt = ShardedOptimizer(base, shards, wire="fp32")
        for k in range(2):
            sopt.zero_grad()
            x, y = data[k][r]
            torch.nn.functional.mse_loss(model(x), y).backward()
            sopt.step()
        return sopt.consolidated_state_dict()

    sd = run_ranks(2, rank_fn)[0]
    assert [g["decoupled_weight_decay"] for g in sd["param_groups"]] == [True, False]
    plain = Adam(_two_groups(make_model(), {}, {}), **BASE[Adam])
    plain.load_state_dict(sd)
    assert [g["decoupled_weight_decay"] for g in plain.param_groups] == [True, False]

    model = make_model()
    base = Adam(_two_groups(model, {}, {}), **BASE[Adam])
    comm = RecordingComm(_Net(1), 0)
    shards = FlatShards(model, comm, wire="fp32", group_of=group_index_of(list(model.parameters()), base))
    sopt = ShardedOptimizer(base, shards, wire="fp32")
    sopt.load_state_dict(sd)
    sopt.zero_grad()
    x, y = data[0][0]
    torch.nn.functional.mse_loss(model(x), y).backward()
    sopt.step()
    assert [a["adamw"] for a in comm.pushed[-1]] == [1, 0] and comm.pushed[-1][0]["step"] == 3

    lin = torch.nn.Linear(4, 3)
    opt = InBackwardOptimizer(Adam(lin.parameters(), decoupled_weight_decay=True, weight_decay=0.1),
                              B200HookState(wire="fp32", total_grad_elems=1))
    opt.step()
    sd1 = opt.state_dict()
    assert sd1["param_groups"][0]["decoupled_weight_decay"] is True
    Adam(torch.nn.Linear(4, 3).parameters()).load_state_dict(sd1)
    params = list(torch.nn.Linear(4, 3).parameters())
    opt2 = InBackwardOptimizer(Adam(params, weight_decay=0.1), B200HookState(wire="fp32", total_grad_elems=1))
    opt2.load_state_dict(sd1)
    flat = torch.zeros(15)
    comm = _FakeComm()
    opt2.apply_bucket(comm, _GradBucket(params, flat), flat, None)
    assert comm.ctx.applied[-1][4].adamw == 1
