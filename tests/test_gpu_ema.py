"""EMA of the weights on one GPU: the fused weight-gradient epilogue and the flat-arena kernel against the reference lerp
bit for bit, the engine over eight steps against the same run without EMA, and a Trainer save / resume round trip."""
import pytest
import torch

from shallowspeed_b200.ops.functional import ema_alpha, ema_lerp_ref

pytestmark = pytest.mark.gpu

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]   # the reference model: cluster chain kernel + grouped wgrad
WIDE = [784, 1024, 640, 10]                       # layer-wise GEMMs (not chain-eligible)
MU, WD = 0.9, 1e-2
ALPHAS = [1.0, ema_alpha(0.999, 1), ema_alpha(0.3, 1)]      # the last one takes the alpha >= 0.5 branch


# ------------------------------------------------------------------ kernel level
# test_gpu_momentum's shapes and test_gpu_gemm's tile edges (k and n across 32 / 64 / 128 boundaries)
SHAPES = [(32, 127, 126), (32, 125, 124), (64, 123, 10), (16, 784, 128), (8, 10, 125), (40, 129, 130), (256, 65, 257)]


def _wgrad(K, dz, x, Wb, Vb, Eb, k, lr, rule, alpha):
    Gb = torch.zeros_like(Wb)
    kw = dict(velocity=Vb[:, :k], momentum=MU, weight_decay=WD) if rule else {}
    if Eb is not None:
        kw.update(ema=Eb[:, :k], ema_alpha=alpha)
    K.linear_wgrad(dz, x, Gb[:, :k], grad_b=Gb[:, k], weight=Wb[:, :k], lr=lr, fuse_sgd=True, precision="fp32", **kw)
    return Gb


@pytest.mark.parametrize("rows,k,n", SHAPES)
@pytest.mark.parametrize("rule", [False, True], ids=["plain", "momentum_wd"])
@pytest.mark.parametrize("alpha", ALPHAS)
def test_fused_wgrad_ema_is_the_reference_lerp(rows, k, n, rule, alpha):
    from shallowspeed_b200.ops import cuda as K

    torch.manual_seed(rows + 3 * k + 7 * n)
    ld = (k + 1 + 7) // 8 * 8
    dz, x = torch.randn(rows, n, device="cuda"), torch.randn(rows, k, device="cuda")
    W0 = torch.zeros(n, ld, device="cuda")
    V0 = torch.zeros(n, ld, device="cuda")
    E0 = torch.zeros(n, ld, device="cuda")
    W0[:, : k + 1] = torch.randn(n, k + 1, device="cuda")
    V0[:, : k + 1] = torch.randn(n, k + 1, device="cuda") * 0.1
    E0[:, : k + 1] = W0[:, : k + 1] + 0.01 * torch.randn(n, k + 1, device="cuda")
    E0[:, k + 1:] = 7.0                                                # padding: must stay as it is
    Wa, Va = W0.clone(), V0.clone()
    _wgrad(K, dz, x, Wa, Va, None, k, 0.05, rule, alpha)              # the same call without EMA
    Wb, Vb, Eb = W0.clone(), V0.clone(), E0.clone()
    Gb = _wgrad(K, dz, x, Wb, Vb, Eb, k, 0.05, rule, alpha)
    torch.cuda.synchronize()
    assert torch.equal(Wb, Wa) and (not rule or torch.equal(Vb, Va))
    assert torch.equal(Eb[:, : k + 1], ema_lerp_ref(E0[:, : k + 1], Wb[:, : k + 1], alpha))
    assert torch.equal(Eb[:, k + 1:], E0[:, k + 1:])
    assert torch.count_nonzero(Gb) == 0
    assert not torch.equal(Wb, W0)                                     # non-vacuous


@pytest.mark.parametrize("n", [1, 7, 4099, 100003])
@pytest.mark.parametrize("rule", [False, True], ids=["plain", "momentum_wd"])
@pytest.mark.parametrize("alpha", ALPHAS)
def test_flat_arena_ema_is_the_reference_lerp(n, rule, alpha):
    from shallowspeed_b200.ops import cuda as K

    torch.manual_seed(n)
    w0, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    v0 = torch.randn(n, device="cuda") * 0.1
    e0 = w0 + 0.01 * torch.randn(n, device="cuda")
    wa, va = w0.clone(), v0.clone()
    if rule:
        K.sgd_momentum_step_(wa, g, va, 0.05, MU, WD, True)
    else:
        K.sgd_step_(wa, g, 0.05)                                       # the plain path the EMA form must round like
    wb, vb, eb = w0.clone(), v0.clone(), e0.clone()
    if rule:
        K.sgd_momentum_step_(wb, g, vb, 0.05, MU, WD, True, ema=eb, ema_alpha=alpha)
    else:
        K.sgd_momentum_step_(wb, g, None, 0.05, 0.0, 0.0, False, ema=eb, ema_alpha=alpha)
    torch.cuda.synchronize()
    assert torch.equal(wb, wa) and (not rule or torch.equal(vb, va))
    assert torch.equal(eb, ema_lerp_ref(e0, wb, alpha))


# ------------------------------------------------------------------ engine level
def _real_mask(arena):
    m = torch.zeros(arena.numel, dtype=torch.bool, device=arena.weights.device)
    for i, (o, k) in enumerate(arena.blocks):
        m[arena.offsets[i]: arena.offsets[i] + o * arena.lds[i]].view(o, arena.lds[i])[:, : k + 1] = True
    return m


def _data(steps, gbs=128):
    from shallowspeed_b200.dataset import synthetic_mnist

    x, y = synthetic_mnist(n=gbs * steps)
    return torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()


@pytest.mark.parametrize("sizes", [SIZES, WIDE], ids=["reference", "wide"])
@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("opt_kw", [{}, dict(momentum=MU, weight_decay=WD)], ids=["plain", "momentum_wd"])
def test_engine_ema_observes_the_run(sizes, precision, opt_kw):
    from shallowspeed_b200.parallel.engine import Trainer

    steps, decay = 8, 0.6
    xh, yh = _data(steps)
    base = Trainer(sizes, lr=0.05, precision=precision, **opt_kw)
    tr = Trainer(sizes, lr=0.05, precision=precision, ema_decay=decay, **opt_kw)
    arena = tr.model.arena
    mask = _real_mask(arena)
    n = arena.numel
    assert torch.equal(tr.model.arena.weights, base.model.arena.weights)
    assert tr.engine.kernels_per_step() == base.engine.kernels_per_step()
    assert "ema=0.6" in tr.engine.describe() and "ema=" not in base.engine.describe()
    e = arena.ema.clone()
    assert torch.equal(e[mask], arena.weights[:n][mask])
    for t in range(steps):
        sl = slice(128 * t, 128 * (t + 1))
        la, lb = base.step(xh[sl], yh[sl]), tr.step(xh[sl], yh[sl])
        assert la == lb
        assert torch.equal(arena.weights, base.model.arena.weights), f"step {t}: the EMA changed the weights"
        if opt_kw:
            assert torch.equal(arena.momentum, base.model.arena.momentum)
        e = torch.where(mask, ema_lerp_ref(e, arena.weights[:n], ema_alpha(decay, t)), e)
        assert torch.equal(arena.ema[mask], e[mask]), f"step {t}: EMA differs from the replayed reference"
        assert not bool(arena.ema[~mask].any())                        # padding stays zero
    assert tr.optimizer.ema_updates == steps
    assert not torch.equal(arena.ema[mask], arena.weights[:n][mask])
    assert torch.equal(tr.ema_state(), arena.ema.cpu())


def test_trainer_save_resume_continues_the_ema_bitwise(tmp_path):
    from shallowspeed_b200.parallel.engine import Trainer
    from shallowspeed_b200.utils.checkpoint import load_stage, save_stage

    kw = dict(momentum=MU, weight_decay=WD, ema_decay=0.9)
    xh, yh = _data(4)
    full = Trainer(SIZES, lr=0.05, **kw)
    for t in range(4):
        full.step(xh[128 * t:128 * (t + 1)], yh[128 * t:128 * (t + 1)])
    part = Trainer(SIZES, lr=0.05, **kw)
    for t in range(2):
        part.step(xh[128 * t:128 * (t + 1)], yh[128 * t:128 * (t + 1)])
    save_stage(part.model, tmp_path, 0, 1, step=2, hparams=kw, momentum=part.worker.optimizer_state(),
               ema=part.ema_state())
    res = Trainer(SIZES, lr=0.05, **kw)
    res.optimizer.ema_updates = load_stage(res.model, tmp_path, 0, 1, expect_hparams=kw)
    for t in range(2, 4):
        res.step(xh[128 * t:128 * (t + 1)], yh[128 * t:128 * (t + 1)])
    assert torch.equal(full.model.arena.weights, res.model.arena.weights)
    assert torch.equal(full.ema_state(), res.ema_state())
    assert not torch.equal(full.ema_state(), full.model.arena.weights[: full.model.arena.numel].cpu())


def test_ema_state_load_roundtrip():
    from shallowspeed_b200.parallel.engine import Trainer

    tr = Trainer(SIZES, lr=0.05, ema_decay=0.9)
    state = tr.ema_state().clone()
    tr.model.arena.ema.zero_()
    tr.worker.load_ema_state(state)
    assert torch.equal(tr.ema_state(), state)
    assert Trainer(SIZES, lr=0.05).ema_state() is None
