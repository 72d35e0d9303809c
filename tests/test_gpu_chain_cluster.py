"""The cluster form of the layer-chain kernel (``csrc/kernels/mlp_chain.cu``): C CTAs per micro-batch, CTA rank c owns
output features [32c, 32c + 32) of every GEMM and the activation panels travel between the CTAs through distributed
shared memory.

CPU: the cluster plan (``chain_cluster_size``, ``chain_cluster_budget``) at every micro-batch size and at the shapes of
``test_gpu_chain.py``.  GPU: the engine runs the expected cluster size, the per-layer fp64 oracle of ``test_gpu_chain.py``
holds for the per-micro-batch and inference launches, and the k-phase reduction is deterministic.
"""
import pytest
import torch

from test_gpu_chain import BASE, SHAPES, _run

REFERENCE = [784, 128, 127, 126, 125, 124, 123, 10]
SMEM_LIMIT = 227 * 1024
# (sizes, C of a training launch: forward + loss head + dgrad chain on the first stage)
EXPECTED_C = [(REFERENCE, 4), (BASE, 4), (SHAPES["c32-k4096"], 3), (SHAPES["depth16"], 2), (SHAPES["straddle-c17"], 1)]


def _layers(sizes):
    return list(zip(sizes[:-1], sizes[1:]))


# ================================================================================================== CPU side
def test_cluster_plan_fits_and_double_buffers_at_every_micro_batch_size():
    from shallowspeed_b200 import _C

    for mb in range(1, 129):
        for split in (False, True):
            assert _C.chain_cluster_budget(mb, 1, split) == _C.chain_budget(mb, split)
            for c in (2, 3, 4):
                ok, kps, stages, smem = _C.chain_cluster_budget(mb, c, split)
                assert ok, (mb, c)
                assert kps in (1, 2, 4) and stages >= 2 and smem <= SMEM_LIMIT, (mb, c, kps, stages, smem)


@pytest.mark.parametrize("sizes,c", EXPECTED_C, ids=["reference", "base", "c32-k4096", "depth16", "straddle-c17"])
def test_cluster_size_follows_the_widths(sizes, c):
    from shallowspeed_b200 import _C

    ly = _layers(sizes)
    #                          fwd    loss   bwd    first  gated  folded
    assert _C.chain_cluster_size(ly, True, True, True, True, False, False) == c             # coalesced training step
    # gated for the LL data-parallel kernel, or folded pipeline boundaries: one CTA per micro-batch
    assert _C.chain_cluster_size(ly, True, True, True, True, True, False) == 1
    assert _C.chain_cluster_size(ly, True, False, False, True, False, True) == 1
    assert _C.chain_cluster_size(ly, False, False, True, True, False, True) == 1


def test_cluster_size_counts_every_tile_the_launch_writes():
    from shallowspeed_b200 import _C

    # inference / forward-only: the forward outputs alone
    assert _C.chain_cluster_size(_layers(BASE), True, True, False, True, False, False) == 4
    assert _C.chain_cluster_size(_layers([784, 64, 10]), True, True, False, True, False, False) == 2
    # backward-only launch: the dgrad outputs (layer 1's input only off the first stage) and the staged dZ_L
    assert _C.chain_cluster_size(_layers([300, 20, 10]), False, False, True, True, False, False) == 1
    assert _C.chain_cluster_size(_layers([60, 20, 10]), False, False, True, False, False, False) == 2
    assert _C.chain_cluster_size(_layers([20, 20, 100]), False, False, True, True, False, False) == 4
    # stages at most 32 wide gain nothing from the split
    assert _C.chain_cluster_size(_layers([784, 32, 32, 10]), True, True, True, True, False, False) == 1


# ================================================================================================== GPU side
def _trainer(sizes, mb_rows, n_mu, precision="fp32"):
    from shallowspeed_b200.parallel.engine import Trainer

    return Trainer(sizes, global_batch_size=mb_rows * n_mu, n_mubatches=n_mu, lr=0.01, precision=precision)


@pytest.mark.gpu
@pytest.mark.parametrize("sizes,c", EXPECTED_C, ids=["reference", "base", "c32-k4096", "depth16", "straddle-c17"])
def test_engine_runs_the_expected_cluster_size(sizes, c):
    tr = _trainer(sizes, 32, 4)
    assert tr.engine.uses_chain()
    assert tr.engine.chain_cluster() == c


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_two_engines_give_bit_identical_weights(precision):
    """The k-phase partial sums are added in a fixed order: two engines on the same inputs agree bit for bit."""
    from shallowspeed_b200.dataset import synthetic_mnist

    x, y = synthetic_mnist(n=128 * 6)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    arenas = []
    for _ in range(2):
        tr = _trainer(REFERENCE, 32, 4, precision)
        assert tr.engine.chain_cluster() == 4
        for i in range(6):
            tr.step_async(xd[i * 128:(i + 1) * 128], yd[i * 128:(i + 1) * 128])
        tr.synchronize()
        arenas.append(tr.model.arena.weights.detach().clone())
    assert bool(torch.isfinite(arenas[0]).all())
    assert torch.equal(arenas[0], arenas[1])


@pytest.mark.gpu
@pytest.mark.parametrize("mb_rows", [24, 40, 100])                      # NTW 2 / 4 / 8
@pytest.mark.parametrize("sizes,c", [(BASE, 4), (SHAPES["c32-k4096"], 3)], ids=["base", "c32-k4096"])
def test_per_micro_batch_launches_with_clusters(sizes, c, mb_rows, monkeypatch):
    """SSB_NO_COALESCE: one forward launch and one backward-only launch (dZ_L staged from global memory) per
    micro-batch, each a cluster of C CTAs."""
    import shallowspeed_b200.parallel.engine as engine_mod

    seen = []

    class Recording(engine_mod.Trainer):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            seen.append(self.engine.chain_cluster())

    monkeypatch.setattr(engine_mod, "Trainer", Recording)
    _run(sizes, mb_rows, 2, "fp32", expect_chain=True, env=("SSB_NO_COALESCE",), monkeypatch=monkeypatch)
    assert seen == [c]


@pytest.mark.gpu
@pytest.mark.parametrize("sizes,mb_rows", [(BASE, 40), (SHAPES["depth16"], 100)], ids=["base", "depth16"])
def test_inference_launch_with_clusters(sizes, mb_rows):
    from shallowspeed_b200.pipe import InferenceSchedule

    tr = _trainer(sizes, mb_rows, 2)
    eng = tr.worker.engine_for(InferenceSchedule(2, 1, 0))
    assert eng.chain_cluster() > 1
    _run(sizes, mb_rows, 2, "fp32", expect_chain=True, inference=True)
