"""SGD momentum / Nesterov / weight decay on the GPU: the fused weight-gradient epilogue and the elementwise kernel
against an fp64 evaluation of the rule, the native engine against the CPU oracle (Python VM), determinism, the
untouched default path and a checkpoint round trip through ``optimizer_state``."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]
MU, WD = 0.9, 1e-2
UPD_TOL = {"tf32": 6e-2, "fp32": 2e-2}       # as tests/test_gpu_engine.py


def _frob(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _rule64(w, g, v, lr, mu, wd, nesterov):
    w, g, v = w.double(), g.double(), v.double()
    gp = g + wd * w
    v = mu * v + gp
    d = gp + mu * v if nesterov else v
    return w - lr * d, v


# ------------------------------------------------------------------ kernel level
@pytest.mark.parametrize("rows,k,n", [(32, 127, 126), (32, 125, 124), (64, 123, 10), (16, 784, 128), (8, 10, 125)])
@pytest.mark.parametrize("wd", [0.0, WD])
@pytest.mark.parametrize("nesterov", [False, True])
def test_fused_wgrad_momentum_matches_fp64(rows, k, n, wd, nesterov):
    from shallowspeed_b200.ops import cuda as K

    torch.manual_seed(rows + 3 * k + 7 * n)
    ld = (k + 1 + 7) // 8 * 8
    dz = torch.randn(rows, n, device="cuda")
    x = torch.randn(rows, k, device="cuda")
    Wb = torch.zeros(n, ld, device="cuda")
    Vb = torch.zeros(n, ld, device="cuda")
    Wb[:, : k + 1] = torch.randn(n, k + 1, device="cuda")
    Vb[:, : k + 1] = torch.randn(n, k + 1, device="cuda") * 0.1
    Gb = torch.zeros(n, ld, device="cuda")
    W0, V0 = Wb.clone(), Vb.clone()
    lr = 0.05
    K.linear_wgrad(dz, x, Gb[:, :k], grad_b=Gb[:, k], weight=Wb[:, :k], lr=lr, fuse_sgd=True, precision="fp32",
                   velocity=Vb[:, :k], momentum=MU, weight_decay=wd, nesterov=nesterov)
    torch.cuda.synchronize()
    g = torch.cat([dz.double().T @ x.double(), dz.double().sum(0, keepdim=True).T], dim=1)
    w_ref, v_ref = _rule64(W0[:, : k + 1], g, V0[:, : k + 1], lr, MU, wd, nesterov)
    dw = Wb[:, : k + 1].double() - W0[:, : k + 1].double()
    assert _frob(dw[:, :k], w_ref[:, :k] - W0[:, :k].double()) < 3e-3
    assert _frob(dw[:, k], w_ref[:, k] - W0[:, k].double()) < 1e-4            # bias column
    assert _frob(Vb[:, : k + 1].double(), v_ref) < 1e-5
    assert torch.count_nonzero(Wb[:, k + 1:]) == 0 and torch.count_nonzero(Vb[:, k + 1:]) == 0   # padding stays zero
    assert torch.count_nonzero(Gb) == 0                                        # dW never touches memory


def test_fused_wgrad_weight_decay_without_momentum():
    from shallowspeed_b200.ops import cuda as K

    torch.manual_seed(5)
    rows, k, n, lr = 32, 127, 126, 0.05
    ld = 128
    dz, x = torch.randn(rows, n, device="cuda"), torch.randn(rows, k, device="cuda")
    Wb = torch.zeros(n, ld, device="cuda")
    Wb[:, : k + 1] = torch.randn(n, k + 1, device="cuda")
    W0, Gb = Wb.clone(), torch.zeros(n, ld, device="cuda")
    K.linear_wgrad(dz, x, Gb[:, :k], grad_b=Gb[:, k], weight=Wb[:, :k], lr=lr, fuse_sgd=True, precision="fp32",
                   weight_decay=WD)
    torch.cuda.synchronize()
    g = torch.cat([dz.double().T @ x.double(), dz.double().sum(0, keepdim=True).T], dim=1)
    # what is left of the update after removing the gradient step must be the decay step -lr * wd * W0, weight tile and
    # bias column alike (a kernel that skips the decay leaves ~0 here)
    decay = Wb[:, : k + 1].double() - W0[:, : k + 1].double() + lr * g
    want = -lr * WD * W0[:, : k + 1].double()
    assert _frob(decay[:, :k], want[:, :k]) < 2e-2
    assert _frob(decay[:, k], want[:, k]) < 2e-2


@pytest.mark.parametrize("n", [1, 7, 4099, 100003])
@pytest.mark.parametrize("mu,wd,nesterov", [(0.9, 0.0, False), (0.9, WD, True), (0.0, WD, False)])
def test_elementwise_momentum_kernel(n, mu, wd, nesterov):
    from shallowspeed_b200.ops import cuda as K

    torch.manual_seed(n)
    w, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    v = torch.randn(n, device="cuda") if mu > 0 else None
    w_ref, v_ref = _rule64(w, g, v if v is not None else torch.zeros_like(w), 0.05, mu, wd, nesterov)
    K.sgd_momentum_step_(w, g, v, 0.05, mu, wd, nesterov)
    torch.cuda.synchronize()
    assert bool(((w.double() - w_ref).abs() <= 1e-6 * (1 + w_ref.abs())).all())
    if v is not None:
        assert bool(((v.double() - v_ref).abs() <= 1e-6 * (1 + v_ref.abs())).all())


# ------------------------------------------------------------------ native engine vs the CPU oracle
def _setup(schedule_cls, steps=1, opt_kw=None, seed_v=True, n_mu=4, lr=0.05, precision="fp32"):
    from shallowspeed_b200.dataset import Dataset, synthetic_mnist
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker
    from shallowspeed_b200.pipe import Worker

    opt_kw = dict(momentum=MU, weight_decay=WD, nesterov=True) if opt_kw is None else opt_kw
    x, y = synthetic_mnist(n=128 * steps)
    v0 = None
    out = {}
    for dev in ("cpu", "cuda"):
        model = MLP(SIZES, 0, 1, 128).to(dev)
        opt = SGD(model.parameters(), lr, arena=model.arena, **opt_kw)
        if seed_v and model.arena.momentum is not None:
            if v0 is None:   # non-zero start on the parameter elements (padding stays 0): one step exercises mu * v
                gen = torch.Generator().manual_seed(3)
                v0 = torch.zeros(model.arena.numel)
                for i, (o, k) in enumerate(model.arena.blocks):
                    off, ld = model.arena.offsets[i], model.arena.lds[i]
                    v0[off:off + o * ld].view(o, ld)[:, : k + 1] = torch.randn(o, k + 1, generator=gen) * 1e-3
            model.arena.momentum.copy_(v0)
        ds = Dataset(None, 128, 128 // n_mu, device=dev)
        ds.local_batch_size = 128
        ds.from_arrays(x, y)
        if dev == "cpu":
            w = Worker(None, None, model, ds, opt)
        else:
            w = NativeWorker(None, None, model, ds, opt, precision=precision)
        for b in range(steps):
            w.execute(schedule_cls(n_mu, 1, 0), b)
        if dev == "cuda":
            w.sync_to_model()
        out[dev] = (model, w)
    return out, v0


ENV_CASES = [{}, {"SSB_NO_CHAIN": "1"}, {"SSB_NO_COALESCE": "1"}, {"SSB_NO_COALESCE": "1", "SSB_NO_CHAIN": "1"}]


@pytest.mark.parametrize("env", ENV_CASES, ids=lambda e: "+".join(sorted(e)) or "default")
@pytest.mark.parametrize("sched", ["naive", "gpipe", "pipedream"])
def test_engine_one_step_with_seeded_momentum(sched, env, monkeypatch):
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.pipe import SCHEDULE_NAME_TO_CLS

    for k, v in env.items():
        monkeypatch.setenv(k, v)
    out, v0 = _setup(SCHEDULE_NAME_TO_CLS[sched])
    (mc, _), (mg, wg) = out["cpu"], out["cuda"]
    init = MLP(SIZES, 0, 1, 128)
    for i, (p0, pc, pg) in enumerate(zip(init.parameters(), mc.parameters(), mg.parameters())):
        err = _frob(pg.data.cpu() - p0.data, pc.data - p0.data)
        assert err < (1e-4 if i % 2 == 1 else 3e-3), (i, err)      # odd = bias, even = weight
    # the momentum buffer's new content minus mu * v0 is the decayed gradient g'
    vc, vg = mc.arena.momentum - MU * v0, mg.arena.momentum.cpu() - MU * v0
    assert _frob(vg, vc) < 3e-3
    # the stateful rule adds no launch
    from shallowspeed_b200.dataset import Dataset
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel.engine import NativeWorker

    plain = MLP(SIZES, 0, 1, 128).to("cuda")
    ds = Dataset(None, 128, 32, device="cuda")
    pw = NativeWorker(None, None, plain, ds, SGD(plain.parameters(), 0.05, arena=plain.arena))
    s = SCHEDULE_NAME_TO_CLS[sched](4, 1, 0)
    assert wg.kernels_per_step(s) == pw.kernels_per_step(s)
    assert "momentum=0.9, nesterov" in wg.describe(s) and "momentum" not in pw.describe(s)


@pytest.mark.parametrize("sched", ["naive", "gpipe", "pipedream"])
def test_engine_three_steps_with_momentum(sched):
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.pipe import SCHEDULE_NAME_TO_CLS

    out, _ = _setup(SCHEDULE_NAME_TO_CLS[sched], steps=3, opt_kw=dict(momentum=MU, weight_decay=1e-3), seed_v=False)
    (mc, _), (mg, wg) = out["cpu"], out["cuda"]
    init = MLP(SIZES, 0, 1, 128)
    for p0, pc, pg in zip(init.parameters(), mc.parameters(), mg.parameters()):
        assert _frob(pg.data.cpu() - p0.data, pc.data - p0.data) < UPD_TOL["fp32"]
    assert wg.kernels_per_step(SCHEDULE_NAME_TO_CLS[sched](4, 1, 0)) == 2


def test_engine_with_momentum_is_bit_deterministic():
    from shallowspeed_b200.pipe import GPipeSchedule

    a = _setup(GPipeSchedule, steps=2)[0]["cuda"][0]
    b = _setup(GPipeSchedule, steps=2)[0]["cuda"][0]
    assert torch.equal(a.arena.weights, b.arena.weights) and torch.equal(a.arena.momentum, b.arena.momentum)


def _trainer_run(steps, **kw):
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer

    x, y = synthetic_mnist(n=128 * steps)
    xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
    tr = Trainer(SIZES, lr=0.05, **kw)
    for i in range(steps):
        tr.step(xh[i * 128:(i + 1) * 128], yh[i * 128:(i + 1) * 128])
    tr.synchronize()
    return tr


def test_default_arguments_keep_the_plain_path_bitwise():
    a = _trainer_run(3)
    b = _trainer_run(3, momentum=0.0, weight_decay=0.0, nesterov=False)
    assert torch.equal(a.model.arena.weights, b.model.arena.weights)
    assert a.engine.kernels_per_step() == b.engine.kernels_per_step() == 2
    assert a.model.arena.momentum is None and b.model.arena.momentum is None
    assert a.engine.plan_text(0) == b.engine.plan_text(0)


def test_engine_refuses_momentum_without_a_buffer():
    from shallowspeed_b200.layers import MLP
    from shallowspeed_b200.optimizer import SGD
    from shallowspeed_b200.parallel import engine as E

    model = MLP(SIZES, 0, 1, 128).to("cuda")
    SGD(model.parameters(), 0.05, momentum=MU, arena=model.arena)
    specs = [(lin.in_dims, lin.out_dims, 1, int(model.arena.offsets[lin.block_index]), int(model.arena.lds[lin.block_index]))
             for lin in model.linears]
    with pytest.raises(RuntimeError, match="momentum buffer"):
        E._C().PipeEngine(specs, dict(momentum=MU), model.arena.weights, model.arena.grads, None)


def test_checkpoint_resume_on_gpu_is_bitwise(tmp_path):
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer
    from shallowspeed_b200.utils.checkpoint import load_stage, save_stage

    kw = dict(momentum=MU, weight_decay=1e-3, nesterov=True)
    x, y = synthetic_mnist(n=128 * 4)
    xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
    batch = lambda i: (xh[i * 128:(i + 1) * 128], yh[i * 128:(i + 1) * 128])
    full = Trainer(SIZES, lr=0.05, **kw)
    for i in range(4):
        full.step(*batch(i))
    full.synchronize()
    part = Trainer(SIZES, lr=0.05, **kw)
    for i in range(2):
        part.step(*batch(i))
    save_stage(part.model, tmp_path, 0, 1, step=2, hparams=kw, momentum=part.worker.optimizer_state())
    res = Trainer(SIZES, lr=0.05, **kw)
    assert load_stage(res.model, tmp_path, 0, 1, expect_hparams=kw) == 2
    state = res.worker.optimizer_state()
    assert torch.equal(state, part.worker.optimizer_state())
    res.worker.load_optimizer_state(state)
    for i in range(2, 4):
        res.step(*batch(i))
    res.synchronize()
    assert torch.equal(full.model.arena.weights, res.model.arena.weights)
    assert torch.equal(full.worker.optimizer_state(), res.worker.optimizer_state())
