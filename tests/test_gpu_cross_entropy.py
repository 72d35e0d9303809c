"""Softmax cross-entropy on the H100: both loss-head kernels (the chain kernel's fused head in its C = 1 and cluster forms,
and ``loss_head_kernel`` of the layer-wise paths) against a per-layer fp64 oracle, the stand-alone op, determinism, the
default (MSE) path, and a short training run against torch in fp64.

The per-layer method is ``test_gpu_chain.py``'s: one training step through ``Trainer``, then every layer on its own from
the engine's buffers, so errors cannot cascade.  The cross-entropy head is checked per micro-batch on the kernel's own
logits, with rtol = 2^-16 (the head is fp32 in both precisions):
    probs  rtol * p
    dz     rtol * p * |T| / B + 3 u |dz|          (T = sum(t); u = 2^-24: three roundings, of fma(p, T, -t), of 1 / B
                                                   and of their product, which is all that remains where p T ~ t)
    loss   rtol * sum_rows sum_k |t_k| (1 + |m - z_k|) / B      (log s is exact to about one ulp)
Worst err / bound over the grid, measured on an H100 80GB HBM3 (400 W): probs 0.076, dz 0.50, loss 0.009; the stand-alone
op dz 0.67 (257 soft-target classes); the layers around the head as in test_gpu_chain.py (tf32 update 0.93).
"""
import math

import pytest
import torch

from test_gpu_chain import (ATOL, HEAD_RTOL, LR, RTOL, _gather, _init_weights, _poison, dgrad_oracle, excess,
                            fwd_oracle, update_oracle)

REFERENCE = [784, 128, 127, 126, 125, 124, 123, 10]
BASE = [784, 128, 97, 33]                   # + the classes: four CTAs per micro-batch
NARROW = [33, 32, 31, 17]                   # every layer at most 32 wide: one CTA per micro-batch
CLASSES = [3, 10, 16, 17, 32]               # fast head up to 16, slow head 17..32
MB_GRID = [1, 8, 24, 32, 100, 128]
UNIT_ROUNDOFF = 2.0**-24


def _n_mu(mb_rows):
    return 1 if mb_rows == 128 else 2


# ================================================================================================== the CE oracle
def ce_head_oracle(z, t, batch, rtol):
    """Cross-entropy head of ONE micro-batch on logits ``z``: (probs, dz, loss) in fp64 (torch's definitions) and their
    bounds."""
    z, t = z.double(), t.double()
    m = z.max(1, keepdim=True).values
    p = torch.softmax(z, -1)
    T = t.sum(1, keepdim=True)
    dz = (p * T - t) / batch
    loss = float(torch.nn.functional.cross_entropy(z, t, reduction="sum")) / batch
    b_p = rtol * p + ATOL
    b_dz = rtol * p * T.abs() / batch + 3.0 * UNIT_ROUNDOFF * dz.abs() + ATOL
    b_loss = rtol * float((t.abs() * (1.0 + (m - z).abs())).sum()) / batch + ATOL
    return (p, b_p), (dz, b_dz), (loss, b_loss)


# ================================================================================================== GPU: one step
def _run_ce(sizes, mb_rows, n_mu, precision, expect_chain, inference=False, env=(), monkeypatch=None, cluster=None):
    """One cross-entropy step at the given shape; returns {check: max err / bound} after asserting the path, the cluster
    size and non-vacuity."""
    from shallowspeed_b200.parallel.engine import Trainer
    from shallowspeed_b200.pipe import InferenceSchedule

    for k in env:
        monkeypatch.setenv(k, "1")
    L, C, rows = len(sizes) - 1, sizes[-1], mb_rows * n_mu
    gen = torch.Generator().manual_seed(hash(("ce", tuple(sizes), mb_rows, n_mu)) & 0xFFFFFFFF)
    x = torch.randn(rows, sizes[0], generator=gen)
    t = torch.nn.functional.one_hot(torch.randint(0, C, (rows,), generator=gen), C).float()
    Ws, bs = _init_weights(sizes, x, n_mu, gen)

    tr = Trainer(sizes, global_batch_size=rows, n_mubatches=n_mu, lr=LR, precision=precision, loss="cross_entropy")
    model = tr.model
    for i, (W, b) in enumerate(zip(Ws, bs)):
        model.arena.weight_view(i).copy_(W)
        model.arena.bias_view(i).copy_(b[None, :])
    if inference:
        sched = InferenceSchedule(n_mu, 1, 0)
        eng = tr.worker.engine_for(sched)
    else:
        eng = tr.engine
    assert eng.uses_chain() == expect_chain
    assert "loss=cross_entropy" in eng.describe()
    if cluster is not None:
        assert eng.chain_cluster() == cluster
    if "SSB_NO_COALESCE" in env:
        assert not eng.coalesced()
    _poison(eng, model, sizes, rows, not inference)
    W0 = [model.arena.block(i)[:, : k + 1].double().cpu() for i, (_, k) in enumerate(model.arena.blocks)]
    xh, th = x.pin_memory(), t.pin_memory()
    if inference:
        tr.worker.step_from(sched, xh, th)
        eng.synchronize()
        loss = None
    else:
        loss = float(tr.step(xh, th))
    torch.cuda.synchronize()

    act = [x.double()] + [_gather(lambda mu, l=l: eng.act(mu, l), n_mu) for l in range(1, L + 1)]
    probs = _gather(eng.probs, n_mu)
    rtol = RTOL[precision]
    res = {}
    for l in range(1, L):
        frac = float((act[l] > 0).double().mean())
        assert 0.05 <= frac <= 0.95, f"layer {l}: {frac:.3f} of the activations are positive"
    for l in range(1, L + 1):
        W, b = W0[l - 1][:, :-1], W0[l - 1][:, -1]
        ref, bound = fwd_oracle(act[l - 1], W, b, l < L, rtol)
        res[f"fwd{l}"] = excess(act[l], ref, bound)
    dz = None
    if not inference:
        dz = [None] + [_gather(lambda mu, l=l: eng.dz(mu, l), n_mu) for l in range(1, L + 1)]
        for l in range(1, L + 1):
            assert float(dz[l].abs().max()) > 0.0, f"dz[{l}] is all zero"
    loss_ref = loss_bound = 0.0
    for mu in range(n_mu):
        r = slice(mu * mb_rows, (mu + 1) * mb_rows)
        (p, bp), (g, bg), (lv, bl) = ce_head_oracle(act[L][r], t[r], rows, HEAD_RTOL)
        res["probs"] = max(res.get("probs", 0.0), excess(probs[r], p, bp))
        if not inference:
            res["dzL"] = max(res.get("dzL", 0.0), excess(dz[L][r], g, bg))
        loss_ref, loss_bound = loss_ref + lv, loss_bound + bl
    if not inference:
        res["loss"] = abs(loss - loss_ref) / loss_bound if math.isfinite(loss) else math.inf
        for l in range(L, 1, -1):
            ref, bound = dgrad_oracle(dz[l], W0[l - 1][:, :-1], act[l - 1], rtol)
            res[f"dgrad{l}"] = excess(dz[l - 1], ref, bound)
        for i, (_, k) in enumerate(model.arena.blocks):
            W1 = model.arena.block(i)[:, : k + 1].double().cpu()
            ref, bound = update_oracle(dz[i + 1], act[i], W0[i], LR, rtol)
            res[f"upd{i + 1}"] = excess(W1 - W0[i], ref, bound)
    worst = max(res, key=res.get)
    print(f"\n[ce] sizes={sizes} mb_rows={mb_rows} n_mu={n_mu} {precision} chain={expect_chain} env={list(env)} "
          f"inference={inference}: max err/bound {res[worst]:.3g} ({worst}); "
          + " ".join(f"{k}={v:.2g}" for k, v in res.items()))
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("mb_rows", MB_GRID)
@pytest.mark.parametrize("classes", CLASSES)
def test_ce_chain_head_classes_and_micro_batch_sizes(classes, mb_rows, precision):
    _run_ce(BASE + [classes], mb_rows, _n_mu(mb_rows), precision, expect_chain=True, cluster=4)


LAUNCH_FORMS = {"coalesced": (), "per-micro-batch": ("SSB_NO_COALESCE",), "layer-wise": ("SSB_NO_CHAIN",),
                "layer-wise-per-micro-batch": ("SSB_NO_COALESCE", "SSB_NO_CHAIN")}


@pytest.mark.gpu
@pytest.mark.parametrize("form", list(LAUNCH_FORMS))
@pytest.mark.parametrize("mb_rows", [24, 100])
@pytest.mark.parametrize("sizes,c", [(BASE + [10], 4), (NARROW, 1), (NARROW[:-1] + [10], 1)],
                         ids=["cluster4-c10", "c1-c17", "c1-c10"])
def test_ce_launch_forms(sizes, c, mb_rows, form, monkeypatch):
    """The cluster (rank 0 runs the head and sends dZ_L) and the C = 1 chain launches, each with the fast head (10
    classes) and the C = 1 one with the slow head (17), per micro-batch as well; the layer-wise forms run
    loss_head_kernel."""
    env = LAUNCH_FORMS[form]
    chain = "SSB_NO_CHAIN" not in env
    _run_ce(sizes, mb_rows, 2, "fp32", expect_chain=chain, env=env, monkeypatch=monkeypatch, cluster=c if chain else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("mb_rows", [24, 128])
def test_ce_more_than_32_classes_runs_layer_wise(mb_rows, precision):
    _run_ce([784, 64, 33], mb_rows, _n_mu(mb_rows), precision, expect_chain=False)


@pytest.mark.gpu
@pytest.mark.parametrize("sizes,mb_rows,chain", [(BASE + [10], 40, True), (NARROW, 100, True), ([784, 64, 33], 24, False)],
                         ids=["cluster4", "c1-c17", "layer-wise-c33"])
def test_ce_inference_probs_are_the_row_softmax(sizes, mb_rows, chain):
    _run_ce(sizes, mb_rows, 2, "fp32", expect_chain=chain, inference=True)


# ================================================================================================== GPU: the op itself
@pytest.mark.gpu
@pytest.mark.parametrize("rows,classes", [(128, 10), (32, 40), (100, 257)], ids=["pp8-last-stage", "c40", "c257"])
@pytest.mark.parametrize("soft", [False, True], ids=["one-hot", "soft"])
def test_ce_loss_head_op(rows, classes, soft):
    """ops.cuda.loss_head_backward / softmax with loss="cross_entropy": the shape the loss-only last stage of pp = 8 runs
    (the whole micro-batch of 10-class logits) and wider heads than the chain takes.  One row lies 200 below the others:
    the global-max contract would lose it."""
    from shallowspeed_b200.ops import cuda as K

    gen = torch.Generator().manual_seed(rows * 1000 + classes)
    z = torch.randn(rows, classes, generator=gen) * 4.0
    z[rows // 2] -= 200.0
    if soft:
        t = torch.rand(rows, classes, generator=gen)
        t = t / t.sum(1, keepdim=True) * 0.75
    else:
        t = torch.nn.functional.one_hot(torch.randint(0, classes, (rows,), generator=gen), classes).float()
    batch = 4 * rows
    dz, p, loss = K.loss_head_backward(z.cuda(), t.cuda(), batch, loss="cross_entropy")
    probs_only = K.softmax(z.cuda(), loss="cross_entropy")
    (pr, bp), (g, bg), (lv, bl) = ce_head_oracle(z, t, batch, HEAD_RTOL)
    res = {"probs": excess(p, pr, bp), "dz": excess(dz, g, bg), "loss": abs(float(loss) - lv) / bl,
           "softmax": excess(probs_only, pr, bp)}
    print(f"\n[ce-op] rows={rows} classes={classes} soft={soft}: " + " ".join(f"{k}={v:.2g}" for k, v in res.items()))
    assert all(v <= 1.0 for v in res.values()), res
    assert torch.equal(probs_only, p)
    with pytest.raises(Exception, match="loss"):
        K.loss_head_backward(z.cuda(), t.cuda(), batch, loss="hinge")


# ================================================================================================== GPU: engines
def _steps(loss, steps=6, sizes=REFERENCE, precision="fp32", lr=0.01, **kw):
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer

    x, y = synthetic_mnist(n=128 * steps)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    tr = Trainer(sizes, global_batch_size=128, n_mubatches=4, lr=lr, precision=precision, **({"loss": loss} if loss else {}),
                 **kw)
    losses = [float(tr.step(xd[i * 128:(i + 1) * 128], yd[i * 128:(i + 1) * 128])) for i in range(steps)]
    return tr, losses


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_ce_engines_are_bit_identical_and_launch_as_many_kernels_as_mse(precision):
    a, la = _steps("cross_entropy", precision=precision)
    b, lb = _steps("cross_entropy", precision=precision)
    assert a.engine.chain_cluster() == 4
    assert la == lb and torch.equal(a.model.arena.weights, b.model.arena.weights)
    assert bool(torch.isfinite(a.model.arena.weights).all())
    mse, _ = _steps("mse", steps=1, precision=precision)
    assert a.engine.kernels_per_step() == mse.engine.kernels_per_step()


@pytest.mark.gpu
def test_default_trainer_is_mse_bitwise():
    a, la = _steps(None)
    b, lb = _steps("mse")
    assert la == lb and torch.equal(a.model.arena.weights, b.model.arena.weights)
    assert "cross_entropy" not in a.engine.describe()


@pytest.mark.gpu
def test_ce_trainer_tracks_torch_fp64():
    """20 steps of the cross-entropy Trainer (fp32 products) against nn.Linear + ReLU + F.cross_entropy in fp64 from the
    same initial weights and batches.  Tolerance: the weights' distance from the fp64 run is below 1e-3 of the distance
    the run moved them, and every step's loss agrees to 1e-4 relative.

    The reference is torch's autograd, not the Python VM: the VM keeps its parameters in an fp32 arena, so it cannot run
    in fp64, and an fp64 torch model does not share any code with the engine under test.  test_cross_entropy.py shows on
    the CPU that the VM matches the same torch model."""
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.layers import MLP

    steps, lr = 20, 0.05
    init = MLP(REFERENCE, 0, 1, 128, loss="cross_entropy")
    ref = [(l._params["W"].data.double().clone().requires_grad_(True),
            l._params["b"].data.reshape(-1).double().clone().requires_grad_(True)) for l in init.linears]
    w0 = torch.cat([torch.cat([W.detach().flatten(), b.detach()]) for W, b in ref])
    tr, losses = _steps("cross_entropy", steps=steps, lr=lr)
    x, y = synthetic_mnist(n=128 * steps)
    ref_losses = []
    for s in range(steps):
        a, t = torch.from_numpy(x[s * 128:(s + 1) * 128]).double(), torch.from_numpy(y[s * 128:(s + 1) * 128]).double()
        for i, (W, b) in enumerate(ref):
            a = a @ W.T + b
            if i < len(ref) - 1:
                a = torch.relu(a)
        loss = torch.nn.functional.cross_entropy(a, t, reduction="sum") / 128
        loss.backward()
        ref_losses.append(float(loss.detach()))
        with torch.no_grad():
            for W, b in ref:
                W -= lr * W.grad
                b -= lr * b.grad
                W.grad, b.grad = None, None
    tr.synchronize()
    got = torch.cat([torch.cat([l._params["W"].data.double().cpu().flatten(), l._params["b"].data.double().cpu().reshape(-1)])
                     for l in tr.model.linears])
    want = torch.cat([torch.cat([W.detach().flatten(), b.detach()]) for W, b in ref])
    moved, err = float((want - w0).norm()), float((got - want).norm())
    rel_loss = max(abs(g - r) / r for g, r in zip(losses, ref_losses))
    print(f"\n[ce-train] moved={moved:.4g} err={err:.3g} ({err / moved:.3g} of it), worst loss rel err {rel_loss:.3g}, "
          f"loss {ref_losses[0]:.4f} -> {ref_losses[-1]:.4f}")
    assert ref_losses[-1] < ref_losses[0]
    assert err < 1e-3 * moved
    assert rel_loss < 1e-4


# ================================================================================================== CPU: the oracle
def test_ce_oracle_rejects_injected_faults():
    """Each fault applied to the exact result is rejected; the exact result and a per-row fp32 evaluation (the kernel's
    contract) are accepted."""
    from shallowspeed_b200.ops import functional as F

    g = torch.Generator().manual_seed(5)
    rows, C, batch = 32, 10, 64
    z = torch.randn(rows, C, generator=g, dtype=torch.float64)
    z = z * (20.0 / float(z.max() - z.min()))                    # the logit spread of the GPU grid
    labels = torch.randint(0, C, (rows,), generator=g)
    labels[0] = int(z[0].argmin())                               # one confidently wrong row
    z[0, labels[0]] = z[0].max() - 25.0
    t = torch.nn.functional.one_hot(labels, C).double()
    (p, bp), (dz, bdz), (loss, bl) = ce_head_oracle(z, t, batch, HEAD_RTOL)

    def ok(pp, gg, ll):
        return excess(pp, p, bp) <= 1.0 and excess(gg, dz, bdz) <= 1.0 and abs(ll - loss) <= bl

    assert ok(p, dz, loss)
    z32, t32 = z.float(), t.float()                              # the kernel's contract evaluated in fp32
    m32 = z32.max(1, keepdim=True).values
    e32 = torch.exp(z32 - m32)
    s32 = e32.sum(1, keepdim=True)
    p32 = e32 / s32
    assert ok(p32, (p32 * t32.sum(1, keepdim=True) - t32) / batch,
              float((t32 * ((m32 - z32) + torch.log(s32))).sum()) / batch)
    # the MSE head's softmax: the micro-batch's max and +1e-7
    pg = F.softmax_ref(z)
    assert not ok(pg, (pg - t) / batch, loss)
    # the MSE gradient through the softmax Jacobian
    assert excess(F.softmax_grad_ref(F.mse_loss_grad_ref(pg, t, batch), z), dz, bdz) > 1.0
    # the 1/B missing, and t - p in place of p - t
    assert excess(dz * batch, dz, bdz) > 1.0
    assert excess(-dz, dz, bdz) > 1.0
    # -log(p + 1e-7) in place of the log-sum-exp
    assert abs(float(-(t * torch.log(p + 1e-7)).sum()) / batch - loss) > bl
