"""The grouped weight-gradient launch on its narrow [32 x 32] tiles against the per-layer kernel (128 x 64 tiles), called
stand-alone, bit for bit, at every tile edge: output features 1, 10, 31, 32, 33, 97, 127, 128, input columns 7, 31, 32,
33, 64, 65, 784, 4096 and 8 to 512 rows (one to sixteen k-blocks, a partial last one), in both precisions and with each
SGD rule.  Each output element goes through the same MMAs, k-block sums, column sum and update in both launches, so after
every step the engine's weights, and the momentum where there is one, must equal what the per-layer kernel makes of the
weights before the step and the step's own dZ and activation rows."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# layer widths; together the three models have each of the edge widths above as a layer's input and as its output (a
# one-class head would have a zero gradient, so the 1-wide layer sits inside a model)
MODELS = [[4096, 128, 33, 64, 127, 10], [784, 97, 65, 31, 1, 32], [7, 128, 7, 32]]
OPTIMIZERS = {"sgd": {}, "momentum_wd": dict(momentum=0.9, weight_decay=5e-4),
              "nesterov": dict(momentum=0.9, weight_decay=5e-4, nesterov=True)}
N_MU, LR, STEPS = 4, 0.05, 3


def _block(flat, arena, i):
    """Block i of a flat buffer laid out like the arena: [out, ld], the bias in column ``in``."""
    out, ld = arena.blocks[i][0], arena.lds[i]
    return flat[arena.offsets[i]: arena.offsets[i] + out * ld].view(out, ld)


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.parametrize("opt", list(OPTIMIZERS))
@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("rows", [8, 24, 100, 128, 512])
@pytest.mark.parametrize("sizes", MODELS, ids=lambda s: "-".join(map(str, s)))
def test_grouped_narrow_tiles_equal_the_stand_alone_per_layer_kernel(sizes, rows, precision, opt):
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.ops import cuda as K
    from shallowspeed_b200.parallel.engine import Trainer

    rule = OPTIMIZERS[opt]
    x, y = synthetic_mnist(n=rows * STEPS, n_features=sizes[0], n_classes=sizes[-1])
    xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
    tr = Trainer(sizes, global_batch_size=rows, n_mubatches=N_MU, lr=LR, precision=precision, seed_mode="index", **rule)
    eng, arena = tr.engine, tr.model.arena
    assert "wgrad_group" in eng.plan_text(0) and " gemm " not in eng.plan_text(0), eng.plan_text(0)
    for step in range(STEPS):
        w0 = arena.weights.clone()
        v0 = arena.momentum.clone() if rule.get("momentum") else None
        run_set = eng.fill_set()                 # the staging set this step's inputs go into
        tr.step(xh[step * rows:(step + 1) * rows], yh[step * rows:(step + 1) * rows])
        tr.synchronize()
        # the per-layer kernel on the weights (and momentum) before the step, fed the step's dZ and activation rows of
        # all micro-batches in micro-batch order; the bias gradient goes to column `in` of a scratch G block
        want_w, want_v = w0.clone(), (v0.clone() if v0 is not None else None)
        for i in range(len(sizes) - 1):
            inp = sizes[i]
            dz = torch.cat([eng.dz(mu, i + 1) for mu in range(N_MU)])
            act = eng.staging(run_set)[0][:, :inp] if i == 0 else torch.cat([eng.act(mu, i) for mu in range(N_MU)])
            w = _block(want_w, arena, i)
            g = torch.empty_like(w)
            v = _block(want_v, arena, i)[:, :inp] if want_v is not None else None
            K.linear_wgrad(dz, act, g[:, :inp], grad_b=g[:, inp], weight=w[:, :inp], lr=LR, fuse_sgd=True,
                           precision=precision, velocity=v, **rule)
        torch.cuda.synchronize()
        assert torch.equal(_bits(arena.weights), _bits(want_w)), f"weights differ after step {step + 1}"
        if v0 is not None:
            assert torch.equal(_bits(arena.momentum), _bits(want_v)), f"momentum differs after step {step + 1}"
