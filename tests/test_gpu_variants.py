"""Kernel variants the engine runs by default:
split-K FWD / DGRAD GEMMs (against an fp64 oracle and the plain kernels, which ``SSB_SPLITK=0`` selects), the zero-copy
loss read-back and the two-node training step of the chain kernel and the grouped weight-gradient launch
(tests/test_gpu_wgrad_group_tiles.py checks that launch bit for bit against the per-layer kernel)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SIZES = [784, 128, 127, 126, 125, 124, 123, 10]


def _report(got, ref, tol):
    """One-glance description of a mismatch (these kernels get few GPU runs: make each one count)."""
    err = (got.double() - ref.double()).abs()
    bad = err > tol
    if not bool(bad.any()):
        return "ok"
    rows = bad.any(1).nonzero().flatten()
    cols = bad.any(0).nonzero().flatten()
    r0, c0 = int(rows[0]), int(cols[0])
    nz = bad & (ref != 0)
    ratio = (got.double()[nz] / ref.double()[nz]).median().item() if bool(nz.any()) else float("nan")
    return (f"max err {err.max().item():.3e} (tol {tol:.1e}); {int(bad.sum())}/{bad.numel()} wrong; rows {int(rows[0])}..{int(rows[-1])} "
            f"({len(rows)} of {got.size(0)}), cols {int(cols[0])}..{int(cols[-1])} ({len(cols)} of {got.size(1)}); "
            f"first bad [{r0},{c0}]: got {got[r0, c0].item():.6g} ref {ref[r0, c0].item():.6g}; median got/ref over bad = {ratio:.4g}; "
            f"zeros in got: {int((got == 0).sum())}, nan: {int(torch.isnan(got).sum())}")


def _rand(*shape, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=torch.float32).cuda()


@pytest.mark.parametrize("precision,tol", [("tf32", 3e-3), ("fp32", 2e-5)])
@pytest.mark.parametrize("rows,inp,out,ks", [(32, 2048, 256, -1), (8, 2048, 200, 3), (128, 4096, 128, 8), (33, 1000, 130, 2)])
def test_splitk_forward_matches_oracle(precision, tol, rows, inp, out, ks):
    from shallowspeed_b200.ops import cuda as K

    x, w, b = _rand(rows, inp, seed=1), _rand(out, inp, seed=2) / inp ** 0.5, _rand(out, seed=3)
    ref = torch.relu(x.double() @ w.double().T + b.double()).float()
    plain = K.linear_fwd(x, w, b, relu=True, precision=precision)[:, :out]
    for _ in range(2):      # each launch allocates fresh counters; tests/test_gpu_gemm.py checks the engine's re-arm
        got = K.linear_fwd(x, w, b, relu=True, precision=precision, k_splits=ks)[:, :out]
        bound = tol * max(ref.abs().max().item(), 1.0) * 4
        assert (got - ref).abs().max().item() <= bound, "vs oracle: " + _report(got, ref, bound)
        assert (got - plain).abs().max().item() <= bound, "vs plain kernel: " + _report(got, plain, bound)


@pytest.mark.parametrize("precision,tol", [("tf32", 3e-3), ("fp32", 2e-5)])
def test_splitk_dgrad_with_relu_mask_matches_oracle(precision, tol):
    from shallowspeed_b200.ops import cuda as K

    rows, inp, out = 32, 300, 4096
    dz, w, act = _rand(rows, out, seed=4), _rand(out, inp, seed=5) / out ** 0.5, _rand(rows, inp, seed=6)
    ref = ((dz.double() @ w.double()) * (act > 0)).float()
    got = K.linear_dgrad(dz, w, mask=act, precision=precision, k_splits=-1)[:, :inp]
    bound = tol * max(ref.abs().max().item(), 1.0) * 4
    assert (got - ref).abs().max().item() <= bound, _report(got, ref, bound)


def test_engine_splitk_trains_like_the_plain_kernels(monkeypatch):
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer

    sizes = [784, 2048, 2048, 10]
    x, y = synthetic_mnist(n=256)
    xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
    monkeypatch.setenv("SSB_SPLITK", "0")
    base = Trainer(sizes, lr=0.05, seed_mode="index")
    assert "splitk_gemms=0" in base.engine.describe()
    ref = [base.step(xh[i * 128:(i + 1) * 128], yh[i * 128:(i + 1) * 128]) for i in range(2)]
    monkeypatch.setenv("SSB_SPLITK", "1")
    tr = Trainer(sizes, lr=0.05, seed_mode="index")
    assert "splitk_gemms=0" not in tr.engine.describe()
    got = [tr.step(xh[i * 128:(i + 1) * 128], yh[i * 128:(i + 1) * 128]) for i in range(2)]
    assert all(abs(a - b) <= 1e-4 * max(1.0, abs(b)) for a, b in zip(got, ref))


# ---------------------------------------------------------------------------------------------------------
# Loss values stored straight into pinned host memory by the loss head: no D2H copy node.
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("env", [{}, {"SSB_NO_CHAIN": "1"}, {"SSB_NO_COALESCE": "1"}])
def test_loss_zero_copy_readback_has_no_copy_node(monkeypatch, env):
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer

    for k, v in env.items():
        monkeypatch.setenv(k, v)
    x, y = synthetic_mnist(n=128 * 4)
    xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
    tr = Trainer(SIZES, lr=0.1)
    assert "loss_d2h" not in tr.engine.plan_text(0) + tr.engine.plan_text(1)
    ref = [tr.step(xh[i * 128:(i + 1) * 128], yh[i * 128:(i + 1) * 128]) for i in range(4)]
    # pipelined read-back: loss of step i is returned by call i + 1
    tr2 = Trainer(SIZES, lr=0.1)
    lag = [tr2.step_pipelined(xh[i * 128:(i + 1) * 128], yh[i * 128:(i + 1) * 128]) for i in range(4)] + [tr2.flush()]
    assert lag[0] is None and lag[1:] == ref


# ---------------------------------------------------------------------------------------------------------
# All layers' weight-gradient tiles in ONE launch behind the chain kernel; with the zero-copy loss the whole step is two
# graph nodes.
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["tf32", "fp32"])
def test_default_training_step_is_a_two_or_three_node_line(precision):
    """chain kernel -> grouped wgrad + SGD in both precisions (3xTF32 derives its lo parts in the kernels): no loss copy
    node, no per-layer fork / join."""
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer
    from shallowspeed_b200.parallel.plan_check import check_plan

    x, y = synthetic_mnist(n=128 * 4)
    xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
    tr = Trainer(SIZES, lr=0.1, precision=precision)
    stats = check_plan(tr.engine.plan_text(0))
    want = 2
    assert stats["kernels_and_copies"] == want, tr.engine.plan_text(0)
    assert int(tr.engine.graph_nodes()) == want
    losses = [tr.step(xh[i * 128:(i + 1) * 128], yh[i * 128:(i + 1) * 128]) for i in range(4)]
    assert all(0.0 < v < 10.0 for v in losses), losses
