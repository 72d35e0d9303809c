"""The grouped weight-gradient launch on its narrow [32 x 32] tiles against the per-layer kernels (SSB_WGRAD_GROUP=0, 128 x 64
tiles), bit for bit, at every tile edge: output features 1, 10, 31, 32, 33, 97, 127, 128, input columns 7, 31, 32, 33, 64,
65, 784, 4096 and 8 to 512 rows (one to sixteen k-blocks, a partial last one), in both precisions and with each SGD rule.
Each output element goes through the same MMAs, k-block sums, column sum and update in both launches, so after three
steps the weights, and the momentum where there is one, must be equal."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# layer widths; together the three models have each of the edge widths above as a layer's input and as its output (a
# one-class head would have a zero gradient, so the 1-wide layer sits inside a model)
MODELS = [[4096, 128, 33, 64, 127, 10], [784, 97, 65, 31, 1, 32], [7, 128, 7, 32]]
OPTIMIZERS = {"sgd": {}, "momentum_wd": dict(momentum=0.9, weight_decay=5e-4),
              "nesterov": dict(momentum=0.9, weight_decay=5e-4, nesterov=True)}


def _train(sizes, rows, precision, opt, group, monkeypatch):
    from shallowspeed_b200.dataset import synthetic_mnist
    from shallowspeed_b200.parallel.engine import Trainer

    monkeypatch.setenv("SSB_WGRAD_GROUP", "1" if group else "0")
    x, y = synthetic_mnist(n=rows * 3, n_features=sizes[0], n_classes=sizes[-1])
    xh, yh = torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory()
    tr = Trainer(sizes, global_batch_size=rows, n_mubatches=4, lr=0.05, precision=precision, seed_mode="index",
                 **OPTIMIZERS[opt])
    assert ("wgrad_group" in tr.engine.plan_text(0)) == group, tr.engine.plan_text(0)
    losses = [tr.step(xh[i * rows:(i + 1) * rows], yh[i * rows:(i + 1) * rows]) for i in range(3)]
    tr.synchronize()
    return tr, losses


@pytest.mark.parametrize("opt", list(OPTIMIZERS))
@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("rows", [8, 24, 100, 128, 512])
@pytest.mark.parametrize("sizes", MODELS, ids=lambda s: "-".join(map(str, s)))
def test_grouped_narrow_tiles_equal_the_per_layer_kernels(monkeypatch, sizes, rows, precision, opt):
    base, ref = _train(sizes, rows, precision, opt, False, monkeypatch)
    tr, got = _train(sizes, rows, precision, opt, True, monkeypatch)
    assert got == ref
    assert torch.equal(tr.model.arena.weights, base.model.arena.weights)
    if OPTIMIZERS[opt].get("momentum"):
        assert torch.equal(tr.model.arena.momentum, base.model.arena.momentum)
