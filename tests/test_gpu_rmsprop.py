"""GPU tests of pose2mesh_release_b200.optim.RMSprop (p2m_rmsprop_step): every element of the parameters and the state
against the float64 restatement within the one-step bound (tests/rmsprop_ref.py), against torch.optim.RMSprop on the
GPU, on the parameter sets of PoseNet and the SMPL-size FlatPose2Mesh with gradients from their native backward, state
dicts in both directions and the reference's resume path, CUDA-graph capture, and determinism."""
import copy

import pytest
import torch

import rmsprop_ref as R
from pose2mesh_release_b200 import _lib
from pose2mesh_release_b200.optim import RMSprop

pytestmark = pytest.mark.gpu

SIZES = (1, 3, 4, 5, 4097, (1 << 20) + 3)
NAMES = {"s": "square_avg", "buf": "momentum_buffer", "ga": "grad_avg"}


def dev():
    return torch.device("cuda:0")


def _grad(gen, n):
    """Gradients over six decades, so that both terms of the bound and every exponent range of s are exercised."""
    return (torch.randn(n, device=dev(), generator=gen) *
            10.0 ** torch.randint(-3, 3, (n,), device=dev(), generator=gen).float())


def _state(opt, p, hp):
    st = opt.state[p]
    out = {"p": p.detach().double(), "s": st["square_avg"].double()}
    if hp["use_momentum"]:
        out["buf"] = st["momentum_buffer"].double()
    if hp["centered"]:
        out["ga"] = st["grad_avg"].double()
    return out


def _ref_step(before, g, hp, err=None):
    return R.step(before["p"], g.double(), before["s"], before.get("buf"), before.get("ga"), hp=hp, err=err)


class _SegmentSet:
    """Two param groups over SIZES: group 0's parameters, gradients and (from the second step) state are views at the
    same odd offsets into flat buffers (16-byte path with scalar heads and tails), group 1's parameters are their own
    allocations with gradients at other offsets (4-byte path).  One parameter of each group never gets a gradient."""

    def __init__(self, opts, lr_tensor, seed=0):
        gen = torch.Generator(device=dev()).manual_seed(seed)
        self.gen = gen
        total = sum(SIZES) + 4 * len(SIZES) + 8
        self.flat = {k: torch.zeros(total, device=dev()) for k in ("p", "g", "s", "buf", "ga")}
        self.flat["p"].copy_(torch.randn(total, device=dev(), generator=gen))
        self.views, off = [], 1
        self.group0 = []
        for n in SIZES:
            self.views.append((off, n))
            self.group0.append(torch.nn.Parameter(self.flat["p"][off:off + n]))
            off += n + 1 + (n % 3)
        self.group1 = [torch.nn.Parameter(torch.randn(n, device=dev(), generator=gen)) for n in SIZES]
        self.g1 = [torch.zeros(n + 2, device=dev())[1 + (i % 2):1 + (i % 2) + n] for i, n in enumerate(SIZES)]
        self.idle = [torch.nn.Parameter(torch.randn(7, device=dev())) for _ in range(2)]
        lrs = (0.01, 0.003)
        lr = [torch.tensor(x, device=dev()) if lr_tensor else x for x in lrs]
        self.opt = RMSprop([{"params": self.group0 + self.idle[:1], "lr": lr[0]},
                            {"params": self.group1 + self.idle[1:], "lr": lr[1]}], alpha=0.9, eps=1e-6, **opts)
        self.hps = [R.fp32_hparams(x, alpha=0.9, eps=1e-6, **opts) for x in lrs]

    def params(self):
        return [(p, 0) for p in self.group0] + [(p, 1) for p in self.group1]

    def set_grads(self):
        for (off, n), p in zip(self.views, self.group0):
            self.flat["g"][off:off + n] = _grad(self.gen, n)
            p.grad = self.flat["g"][off:off + n]
        for p, g in zip(self.group1, self.g1):
            g.copy_(_grad(self.gen, g.numel()))
            p.grad = g

    def share_state(self):
        """Group 0's state as views into flat buffers at its parameters' offsets (values kept)."""
        for (off, n), p in zip(self.views, self.group0):
            st = self.opt.state[p]
            for k, name in NAMES.items():
                if name in st:
                    view = self.flat[k][off:off + n]
                    view.copy_(st[name])
                    st[name] = view


@pytest.mark.parametrize("lr_tensor", (False, True), ids=("lr_float", "lr_tensor"))
@pytest.mark.parametrize("opts", R.OPTION_GRID, ids=lambda o: "wd{weight_decay}-mu{momentum}-c{centered:d}".format(**o))
def test_every_element_within_one_step_bound(opts, lr_tensor):
    """50 steps, each from the device's own previous state: every element of p and of the state within the bound of
    one fp32 step from exact inputs; parameters without a gradient untouched and without state."""
    seg = _SegmentSet(opts, lr_tensor)
    idle = [p.detach().clone() for p in seg.idle]
    for k in range(50):
        seg.set_grads()
        before = [(_state(seg.opt, p, seg.hps[gi]) if k else None, p.grad.clone(), p, gi) for p, gi in seg.params()]
        seg.opt.step()
        torch.cuda.synchronize()
        if k == 0:
            seg.share_state()
            continue
        for b, g, p, gi in before:
            ref, bound = _ref_step(b, g, seg.hps[gi])
            got = _state(seg.opt, p, seg.hps[gi])
            for key in ref:
                bad = R.exceed(got[key], ref[key], bound[key])
                assert bad == 0, (k, p.numel(), gi, key, bad)
            assert seg.opt.state[p]["step"].item() == k + 1
    for p, p0 in zip(seg.idle, idle):
        assert torch.equal(p.detach(), p0) and len(seg.opt.state[p]) == 0


def _pair(params, opts, lr=0.01):
    """A native and a torch optimizer over two copies of `params` (lists of float32 CUDA tensors)."""
    a = [torch.nn.Parameter(t.detach().clone()) for t in params]
    b = [torch.nn.Parameter(t.detach().clone()) for t in params]
    return a, RMSprop(a, lr=lr, **opts), b, torch.optim.RMSprop(b, lr=lr, foreach=True, **opts)


def _accumulated(exact, grads, hp, err):
    """The exact trajectory's next state and the accumulated bound, per tensor."""
    out = []
    for ex, g, e in zip(exact, grads, err):
        ref, bound = _ref_step(ex, g, hp, e)
        out.append((ref, bound))
    return [o[0] for o in out], [o[1] for o in out]


def _start(ps, hp):
    z = lambda p: torch.zeros_like(p, dtype=torch.float64)
    out = []
    for p in ps:
        d = {"p": p.detach().double(), "s": z(p)}
        if hp["use_momentum"]:
            d["buf"] = z(p)
        if hp["centered"]:
            d["ga"] = z(p)
        out.append(d)
    return out


def _check_pair(opt_a, pa, opt_b, pb, exact, err, hp, what):
    for a, b, ex, e in zip(pa, pb, exact, err):
        ga, gb = _state(opt_a, a, hp), _state(opt_b, b, hp)
        for key in ex:
            assert R.exceed(ga[key], gb[key].double(), 2 * e[key]) == 0, (what, a.numel(), key)


@pytest.mark.parametrize("opts", R.OPTION_GRID, ids=lambda o: "wd{weight_decay}-mu{momentum}-c{centered:d}".format(**o))
def test_against_torch_for_100_steps(opts):
    """Same start, same gradients for 100 steps: native and torch's foreach RMSprop differ by at most twice the bound
    accumulated along the exact trajectory (each step's bound taken with the previous step's as input bounds)."""
    gen = torch.Generator(device=dev()).manual_seed(3)
    shapes = [(4097,), (64, 51), (3,), (1 << 16) + 1]
    params = [torch.randn(s, device=dev(), generator=gen) for s in shapes]
    pa, oa, pb, ob = _pair(params, opts)
    hp = R.fp32_hparams(0.01, **opts)
    exact, err = _start(pa, hp), [None] * len(pa)
    bitwise = True
    for k in range(100):
        grads = [_grad(gen, p.numel()).reshape(p.shape) for p in pa]
        for a, b, g in zip(pa, pb, grads):
            a.grad, b.grad = g.clone(), g.clone()
        oa.step()
        ob.step()
        exact, err = _accumulated(exact, grads, hp, err)
        _check_pair(oa, pa, ob, pb, exact, err, hp, k)
        bitwise = bitwise and all(torch.equal(a, b) for a, b in zip(pa, pb))
    assert all(oa.state[a]["step"].item() == 100 for a in pa)
    print(f"RMSprop {opts}: native bitwise equal to torch's foreach path over 100 steps: {bitwise}")


def test_non_finite_gradients_behave_as_torchs():
    """A NaN gradient element makes that parameter NaN in both; a gradient whose square overflows leaves the parameter
    unchanged (g / inf = 0) in both; everything else agrees within the bound."""
    gen = torch.Generator(device=dev()).manual_seed(5)
    pa, oa, pb, ob = _pair([torch.randn(1000, device=dev(), generator=gen)], {})
    g = torch.randn(1000, device=dev(), generator=gen)
    g[7], g[400] = float("nan"), 1e30
    p0 = pa[0].detach().clone()
    pa[0].grad, pb[0].grad = g.clone(), g.clone()
    oa.step()
    ob.step()
    a, b = pa[0].detach(), pb[0].detach()
    assert torch.equal(a.isnan(), b.isnan()) and a.isnan().nonzero().flatten().tolist() == [7]
    assert a[400] == b[400] == p0[400] and oa.state[pa[0]]["square_avg"][400].isinf()
    hp = R.fp32_hparams(0.01)
    ref, bound = _ref_step(_start(pa, hp)[0] | {"p": p0.double()}, g, hp)
    ok = g.isfinite() & (g.abs() < 1e18)
    assert R.exceed(a[ok], ref["p"][ok], bound["p"][ok]) == 0


# ---- the real parameter sets


def _posenet():
    from pose2mesh_release_b200 import posenet

    torch.manual_seed(0)
    net = posenet.get_model(17, 4096, 2, 0.5).to(dev()).train()
    x = torch.randn(64, 34, device=dev())

    def loss():
        return net(x).abs().mean()

    return net, loss


def _flat_pose2mesh():
    from pose2mesh_release_b200 import graph as pg
    from pose2mesh_release_b200.pose2mesh_net import FlatPose2Mesh

    face = pg.synthetic_sphere_faces(6890, 2)
    _, graph_L, _, _ = pg.build_coarse_graphs(face, 17, pg.H36M_SKELETON, pg.H36M_FLIP_PAIRS, levels=9)
    torch.manual_seed(0)
    model = FlatPose2Mesh(17, graph_L).to(dev()).train()
    g = torch.Generator(device=dev()).manual_seed(1)
    pose2d = torch.randn(16, 17, 2, device=dev(), generator=g)
    tgt = torch.randn(16, model.pose2mesh.num_vertices, 3, device=dev(), generator=g)

    def loss():
        mesh, pose3d = model(pose2d)
        return (mesh - tgt).abs().mean() + pose3d.abs().mean()

    return model, loss


@pytest.mark.parametrize("build,n_tensors", ((_posenet, 20), (_flat_pose2mesh, 104)), ids=("posenet", "flat_pose2mesh"))
def test_real_parameter_sets_against_torch(build, n_tensors):
    """Gradients from the native backward fed to both optimizers for 3 steps: within twice the accumulated bound; one
    launch per step for the whole set (22 and 106 tensors); parameters without a gradient (PoseNet's unused
    batch_norm1) get no state."""
    model, loss = build()
    opt = RMSprop(model.parameters(), lr=1e-3)
    named = list(model.named_parameters())
    twins = [torch.nn.Parameter(p.detach().clone()) for _, p in named]
    ref = torch.optim.RMSprop(twins, lr=1e-3)
    hp = R.fp32_hparams(1e-3)
    exact, err = _start([p for _, p in named], hp), [None] * len(named)
    lib = _lib.load()
    for k in range(3):
        model.zero_grad(set_to_none=True)
        loss().backward()
        stepped = [(i, p) for i, (_, p) in enumerate(named) if p.grad is not None]
        assert len(stepped) == n_tensors
        for i, p in stepped:
            twins[i].grad = p.grad.clone()
        lib.p2m_launch_count_reset()
        opt.step()
        assert lib.p2m_launch_count() == 1
        ref.step()
        sub = lambda xs: [xs[i] for i, _ in stepped]
        new_exact, new_err = _accumulated(sub(exact), [p.grad for _, p in stepped], hp, sub(err))
        for (i, _), ex, e in zip(stepped, new_exact, new_err):
            exact[i], err[i] = ex, e
        _check_pair(opt, [p for _, p in stepped], ref, sub(twins), new_exact, new_err, hp, k)
    for name, p in named:
        assert (len(opt.state[p]) == 0) == (p.grad is None), name


# ---- state dicts


def _run(opt, params, grads):
    for g in grads:
        for p, gp in zip(params, g):
            p.grad = gp.clone()
        opt.step()


def _grads(n_steps, shapes, seed):
    gen = torch.Generator(device=dev()).manual_seed(seed)
    return [[_grad(gen, int(torch.tensor(s).prod())).reshape(s) for s in shapes] for _ in range(n_steps)]


@pytest.mark.parametrize("opts", [dict(), dict(momentum=0.9, centered=True, weight_decay=1e-3)])
def test_state_dicts_in_both_directions_and_the_resume_path(opts):
    """torch -> native -> continue, native -> torch -> continue and the reference's resume path (load on the CPU, move
    the state with .cuda(), step) agree with an uninterrupted native run within twice the accumulated bound."""
    shapes = [(51,), (300, 7), (4099,)]
    gen = torch.Generator(device=dev()).manual_seed(9)
    start = [torch.randn(s, device=dev(), generator=gen) for s in shapes]
    grads = _grads(6, shapes, 11)
    hp = R.fp32_hparams(0.01, **opts)
    exact, err = _start(start, hp), [None] * len(start)
    for g in grads:
        exact, err = _accumulated(exact, g, hp, err)

    base = [torch.nn.Parameter(t.clone()) for t in start]
    uninterrupted = RMSprop(base, lr=0.01, **opts)
    _run(uninterrupted, base, grads)

    def check(opt, params, what):
        _check_pair(opt, params, uninterrupted, base, exact, err, hp, what)

    # torch for 3 steps -> native for 3
    pt = [torch.nn.Parameter(t.clone()) for t in start]
    first = torch.optim.RMSprop(pt, lr=0.01, **opts)
    _run(first, pt, grads[:3])
    second = RMSprop(pt, lr=0.01, **opts)
    second.load_state_dict(first.state_dict())
    _run(second, pt, grads[3:])
    check(second, pt, "torch -> native")
    assert all(second.state[p]["step"].item() == 6 and second.state[p]["step"].is_cuda for p in pt)

    # native for 3 steps -> torch for 3
    pn = [torch.nn.Parameter(t.clone()) for t in start]
    first = RMSprop(pn, lr=0.01, **opts)
    _run(first, pn, grads[:3])
    second = torch.optim.RMSprop(pn, lr=0.01, **opts)
    second.load_state_dict(first.state_dict())
    _run(second, pn, grads[3:])
    check(second, pn, "native -> torch")

    # the reference's resume path (lib/core/base.py:62-77, 107): CPU model and optimizer, checkpoint loaded on the CPU,
    # state moved with .cuda(), the model moved afterwards, then steps
    pr = [torch.nn.Parameter(t.clone()) for t in start]
    first = RMSprop(pr, lr=0.01, **opts)
    _run(first, pr, grads[:3])
    ckpt = {"model": [p.detach().cpu() for p in pr], "optim": copy.deepcopy(first.state_dict())}
    ckpt["optim"]["state"] = {i: {k: v.cpu() for k, v in st.items()} for i, st in ckpt["optim"]["state"].items()}
    model = torch.nn.ParameterList([torch.nn.Parameter(torch.zeros(s)) for s in shapes])
    resumed = RMSprop(model.parameters(), lr=0.01, **opts)
    for p, v in zip(model, ckpt["model"]):
        p.data.copy_(v)
    resumed.load_state_dict(ckpt["optim"])
    for state in resumed.state.values():
        for k, v in state.items():
            if torch.is_tensor(v):
                state[k] = v.cuda()
    model = model.cuda()
    _run(resumed, list(model), grads[3:])
    check(resumed, list(model), "resume")


# ---- capture and determinism


def test_captured_step_replays_across_a_milestone():
    """step() with a tensor lr captured once and replayed under MultiStepLR (milestones 3 and 5) is bitwise the eager
    native run with the same lr sequence, step counters included."""
    shapes = [(4097,), (51,), (300, 7)]
    gen = torch.Generator(device=dev()).manual_seed(2)
    start = [torch.randn(s, device=dev(), generator=gen) for s in shapes]
    grads = _grads(8, shapes, 4)

    def make():
        ps = [torch.nn.Parameter(t.clone()) for t in start]
        opt = RMSprop(ps, lr=torch.tensor(0.01, device=dev()), momentum=0.5)
        return ps, opt, torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[3, 5], gamma=0.1)

    pe, oe, se = make()
    for g in grads:
        _run(oe, pe, [g])
        se.step()

    pg, og, sg = make()
    static = [torch.zeros(s, device=dev()) for s in shapes]
    for p, s in zip(pg, static):
        p.grad = s
    for s, g in zip(static, grads[0]):
        s.copy_(g)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                       # the first step eagerly: it creates the state
        og.step()
    torch.cuda.current_stream().wait_stream(side)
    sg.step()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        og.step()
    for g in grads[1:]:
        for s, gi in zip(static, g):
            s.copy_(gi)
        graph.replay()
        sg.step()
    torch.cuda.synchronize()
    for a, b in zip(pe, pg):
        assert torch.equal(a, b)
        for k in ("step", "square_avg", "momentum_buffer"):
            assert torch.equal(oe.state[a][k], og.state[b][k]), k
    assert og.state[pg[0]]["step"].item() == 8 and abs(og.param_groups[0]["lr"].item() - 1e-4) < 1e-10


def test_captured_posenet_training_step_replays():
    """Native PoseNet forward + backward + RMSprop step captured once: 4 replays are bitwise 4 eager steps."""
    from pose2mesh_release_b200 import posenet

    torch.manual_seed(0)
    net_e = posenet.get_model(17, 1024, 1, 0.5).to(dev()).train()
    net_g = copy.deepcopy(net_e)
    gen = torch.Generator(device=dev()).manual_seed(6)
    x, d_out = torch.randn(64, 34, device=dev(), generator=gen), torch.randn(64, 51, device=dev(), generator=gen)
    seed = torch.tensor([3, 1], dtype=torch.int64, device=dev())

    def trained(net):
        return [p for p in net.parameters() if p is not net.batch_norm1.weight and p is not net.batch_norm1.bias]

    def train_step(net, opt):
        params = trained(net)
        grads = torch.autograd.grad(net.forward_train_native(x, seed=seed), params, d_out)
        for p, g in zip(params, grads):
            p.grad = g
        opt.step()

    opt_e = RMSprop(net_e.parameters(), lr=torch.tensor(1e-3, device=dev()))
    for _ in range(5):
        train_step(net_e, opt_e)

    opt_g = RMSprop(net_g.parameters(), lr=torch.tensor(1e-3, device=dev()))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        train_step(net_g, opt_g)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        train_step(net_g, opt_g)
    for _ in range(4):
        graph.replay()
    torch.cuda.synchronize()
    for (k, a), b in zip(net_e.state_dict().items(), net_g.state_dict().values()):
        assert torch.equal(a, b), k
    assert opt_g.state[net_g.w1.weight]["step"].item() == 5


def test_two_runs_are_bitwise_equal():
    seg_a = _SegmentSet(dict(momentum=0.9, centered=True, weight_decay=0.01), True, seed=8)
    seg_b = _SegmentSet(dict(momentum=0.9, centered=True, weight_decay=0.01), True, seed=8)
    for seg in (seg_a, seg_b):
        for _ in range(5):
            seg.set_grads()
            seg.opt.step()
    for (a, _), (b, _) in zip(seg_a.params(), seg_b.params()):
        assert torch.equal(a, b)
        for k in ("square_avg", "momentum_buffer", "grad_avg"):
            assert torch.equal(seg_a.opt.state[a][k], seg_b.opt.state[b][k])
