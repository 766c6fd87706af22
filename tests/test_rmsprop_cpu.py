"""The RMSprop optimizer without a GPU: the float64 restatement (tests/rmsprop_ref.py) against torch.optim.RMSprop in
float64, construction and state-dict layout of pose2mesh_release_b200.optim.RMSprop on CPU parameters, and
install(replace_optimizer=True) over stand-ins of the reference's funcs_utils and core.base."""
import sys
import types

import pytest
import torch

import rmsprop_ref as R
from pose2mesh_release_b200.optim import RMSprop


@pytest.mark.parametrize("foreach", (False, True))
@pytest.mark.parametrize("opts", R.OPTION_GRID, ids=lambda o: "wd{weight_decay}-mu{momentum}-c{centered:d}".format(**o))
def test_restatement_matches_torch_in_float64(opts, foreach):
    """20 steps of torch's float64 RMSprop, each taken from torch's own state, agree with the restatement within twice
    the float64 bound (both round: the restatement once per operation, torch in its own order)."""
    gen = torch.Generator().manual_seed(1)
    n = 2000
    p = torch.nn.Parameter(torch.randn(n, dtype=torch.float64, generator=gen))
    opt = torch.optim.RMSprop([p], lr=0.01, alpha=0.9, eps=1e-6, foreach=foreach, **opts)
    hp = R.f64_hparams(0.01, alpha=0.9, eps=1e-6, **opts)
    names = {"s": "square_avg", "buf": "momentum_buffer", "ga": "grad_avg"}
    zero = torch.zeros(n, dtype=torch.float64)
    before = {"p": p.detach().clone(), "s": zero, "buf": zero, "ga": zero}
    for k in range(20):
        g = torch.randn(n, dtype=torch.float64, generator=gen) * 10.0 ** torch.randint(-4, 4, (n,), generator=gen)
        p.grad = g.clone()
        opt.step()
        ref, bound = R.step(before["p"], g, before["s"], before["buf"], before["ga"], hp=hp, u=R.U64, eta=R.ETA64)
        got = {"p": p.detach()}
        got.update({k2: opt.state[p][names[k2]] for k2 in ref if k2 != "p"})
        for key in ref:
            assert R.exceed(got[key], ref[key], 2 * bound[key]) == 0, (k, key)
        before.update({key: t.clone() for key, t in got.items()})


def test_construction_on_cpu_and_step_needs_cuda():
    lin = torch.nn.Linear(4, 3)
    opt = RMSprop(lin.parameters(), lr=1e-3)
    lin(torch.randn(2, 4)).sum().backward()
    with pytest.raises(RuntimeError, match="contiguous float32 CUDA"):
        opt.step()
    assert len(opt.state) == 0
    for bad in (dict(maximize=True), dict(differentiable=True)):
        with pytest.raises(ValueError, match="not implemented"):
            RMSprop(lin.parameters(), **bad)
    for bad in (dict(lr=-1.0), dict(alpha=-0.5), dict(eps=-1.0), dict(momentum=-0.1), dict(weight_decay=-1.0)):
        with pytest.raises(ValueError, match="Invalid"):
            RMSprop(lin.parameters(), **bad)
    with pytest.raises(ValueError, match="1-element"):
        RMSprop(lin.parameters(), lr=torch.tensor([1e-3, 1e-3]))


@pytest.mark.parametrize("opts", [dict(), dict(momentum=0.5, centered=True, weight_decay=1e-4, alpha=0.9)])
def test_state_dict_layout_is_torchs(opts):
    """Param groups carry torch's keys and values; a stepped torch state loads into the native optimizer and comes back
    out unchanged (keys, shapes, dtypes, values), and loads back into torch."""
    def model():
        torch.manual_seed(0)
        return torch.nn.Sequential(torch.nn.Linear(5, 7), torch.nn.ReLU(), torch.nn.Linear(7, 2))

    m_t, m_n = model(), model()
    ref = torch.optim.RMSprop(m_t.parameters(), lr=1e-3, **opts)
    nat = RMSprop(m_n.parameters(), lr=1e-3, **opts)
    assert nat.state_dict() == ref.state_dict()
    m_t[0].weight.grad = torch.randn(7, 5)            # the other tensors have no gradient: no state
    m_t[2].bias.grad = torch.randn(2)
    ref.step()
    sd = ref.state_dict()
    nat.load_state_dict(sd)
    out = nat.state_dict()
    assert out["param_groups"] == sd["param_groups"] and sorted(out["state"]) == sorted(sd["state"]) == [0, 3]
    for i, st in sd["state"].items():
        assert sorted(out["state"][i]) == sorted(st)
        for k, v in st.items():
            w = out["state"][i][k]
            assert w.shape == v.shape and w.dtype == v.dtype and torch.equal(w, v), (i, k)
    back = torch.optim.RMSprop(model().parameters(), lr=1e-3, **opts)
    back.load_state_dict(out)
    assert back.state_dict()["param_groups"] == sd["param_groups"]


# ---- install(replace_optimizer=True)


def _stand_in_funcs_utils():
    """funcs_utils with its own cfg global and get_optimizer (lib/funcs_utils.py:78-99), and core.base holding the
    function by `from funcs_utils import get_optimizer` (lib/core/base.py:17)."""
    fu = types.ModuleType("funcs_utils")
    fu.cfg = types.SimpleNamespace(TRAIN=types.SimpleNamespace(optimizer="rmsprop", lr=1e-3))
    fu.optim, fu.returned = torch.optim, []
    exec("def get_optimizer(model):\n"
         "    if cfg.TRAIN.optimizer == 'sgd':\n"
         "        opt = optim.SGD(model.parameters(), lr=cfg.TRAIN.lr)\n"
         "    elif cfg.TRAIN.optimizer == 'rmsprop':\n"
         "        opt = optim.RMSprop(model.parameters(), lr=cfg.TRAIN.lr)\n"
         "    else:\n"
         "        opt = optim.Adam(model.parameters(), lr=cfg.TRAIN.lr)\n"
         "    returned.append(opt)\n"
         "    return opt\n", fu.__dict__)
    core = types.ModuleType("core")
    core.__path__ = []
    base = types.ModuleType("core.base")
    base.get_optimizer = fu.get_optimizer
    core.base = base
    return {"funcs_utils": fu, "core": core, "core.base": base}


@pytest.fixture()
def reference():
    from test_install_cpu import _stand_in_reference

    mods = {**_stand_in_reference(), **_stand_in_funcs_utils()}
    saved = {name: sys.modules.get(name) for name in mods}
    sys.modules.update(mods)
    import pose2mesh_release_b200.install as inst

    try:
        yield mods["funcs_utils"], mods["core.base"], inst
    finally:
        inst.uninstall()
        for name, mod in saved.items():
            if mod is None:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = mod


def test_install_replace_optimizer_rebinds_and_uninstall_restores(reference):
    fu, base, inst = reference
    orig = fu.get_optimizer
    model = torch.nn.Linear(3, 2)
    inst.install()                                          # the default leaves the optimizer alone
    assert fu.get_optimizer is orig and base.get_optimizer is orig
    inst.uninstall()
    inst.install(replace_optimizer=True)
    assert fu.get_optimizer is not orig and base.get_optimizer is fu.get_optimizer
    opt = base.get_optimizer(model=model)
    assert type(opt) is RMSprop and opt.defaults == torch.optim.RMSprop(model.parameters(), lr=1e-3).defaults
    assert fu.returned == []
    for name in ("sgd", "adam"):
        fu.cfg.TRAIN.optimizer = name
        got = base.get_optimizer(model=model)
        assert got is fu.returned[-1] and type(got) is {"sgd": torch.optim.SGD, "adam": torch.optim.Adam}[name]
    inst.install(replace_optimizer=True)                    # idempotent
    inst.uninstall()
    assert fu.get_optimizer is orig and base.get_optimizer is orig
