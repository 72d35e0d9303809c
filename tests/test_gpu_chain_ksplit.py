"""The k-split first layer of the cluster chain kernel (``csrc/kernels/mlp_chain.cu``): a cluster launch whose layer 1
has more than 4 k-blocks runs two CTAs per feature slice, the owner multiplying the k-blocks kb with kb % 4 in {0, 1}
and the helper those in {2, 3}.

CPU: the partition of the k-blocks and the shared-memory plan.  GPU: the engines run the k-split where it applies and
only there, and the per-layer fp64 oracles of ``test_gpu_chain.py``, ``test_gpu_cross_entropy.py`` and
``test_gpu_dropout.py`` hold at first-layer widths that end inside a group of four k-blocks.
"""
import pytest
import torch

from test_gpu_chain import BASE, SHAPES, _run

REFERENCE = [784, 128, 127, 126, 125, 124, 123, 10]
SMEM_LIMIT = 227 * 1024
WIDTHS = [129, 160, 200]                  # 5, 5 and 7 k-blocks: the last group of four ends in either part
HIDDEN = BASE[1:]                         # [128, 97, 33, 10]: four CTAs per feature slice set


def _sizes(k):
    return [k] + HIDDEN


# ================================================================================================== CPU side
@pytest.mark.parametrize("k", [129, 160, 200, 784, 4096])
def test_partition_covers_every_kblock_once_in_order(k):
    from shallowspeed_b200 import _C

    nkb = (k + 31) // 32
    parts = [_C.chain_ksplit_kblocks(nkb, part) for part in (0, 1)]
    assert sorted(parts[0] + parts[1]) == list(range(nkb))
    for part, kbs in enumerate(parts):
        assert kbs == sorted(kbs)                                   # increasing, so each k-phase is in k-block order
        # the kernel sums the i-th k-block of a part into the accumulator of k-phase 2 part + (i & 1)
        assert all(kb % 4 == 2 * part + (i & 1) for i, kb in enumerate(kbs)), (part, kbs)
    assert len(parts[0]) - len(parts[1]) in (0, 1, 2)


def test_cluster_budget_fits_at_every_micro_batch_size():
    from shallowspeed_b200 import _C

    for mb in range(1, 129):
        n_pad = (mb + 15) // 16 * 16
        for split in (False, True):
            for c in (2, 3, 4):
                ok, kps, stages, smem = _C.chain_cluster_budget(mb, c, split)
                assert ok, (mb, c)
                assert kps in (1, 2, 4) and stages >= 2 and smem <= SMEM_LIMIT, (mb, c, kps, stages, smem)
                # the ring, the activation ping-pong, the landing area of the helper and the loss head's scratch
                ring = stages * kps * (32 * 128 + n_pad * 128)
                assert smem >= ring + 2 * 4 * n_pad * 128 + 256 * n_pad + n_pad * 33 * 4, (mb, c, smem)


# ================================================================================================== GPU side
def _trainer(sizes, mb_rows, n_mu, **kw):
    from shallowspeed_b200.parallel.engine import Trainer

    return Trainer(sizes, global_batch_size=mb_rows * n_mu, n_mubatches=n_mu, lr=0.01, **kw)


@pytest.mark.gpu
def test_reference_model_runs_two_ctas_per_slice():
    tr = _trainer(REFERENCE, 32, 4)
    assert tr.engine.uses_chain()
    assert tr.engine.chain_cluster() == 4
    assert tr.engine.chain_ksplit() == 2


@pytest.mark.gpu
@pytest.mark.parametrize("sizes,c", [(SHAPES["depth16"], 2), ([128, 128, 97, 33, 10], 4), (SHAPES["straddle-c17"], 1),
                                     ([784, 32, 24, 10], 1)],
                         ids=["k100", "k128", "narrow", "one-cta-k784"])
def test_no_ksplit_where_layer_1_is_short_or_one_cta_owns_the_micro_batch(sizes, c):
    tr = _trainer(sizes, 32, 4)
    assert tr.engine.uses_chain()
    assert tr.engine.chain_cluster() == c
    assert tr.engine.chain_ksplit() == 1


def test_gated_and_folded_launches_run_one_cta():
    """Gated and folded launches run one CTA per micro-batch (C = 1), and a k-split needs C > 1."""
    from shallowspeed_b200 import _C

    ly = list(zip(REFERENCE[:-1], REFERENCE[1:]))
    #                          fwd    loss   bwd    first  gated  folded
    assert _C.chain_cluster_size(ly, True, True, True, True, True, False) == 1
    assert _C.chain_cluster_size(ly, True, False, False, True, False, True) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("mb_rows", [24, 40, 100])                      # NTW 2 / 4 / 8
@pytest.mark.parametrize("k", WIDTHS)
@pytest.mark.parametrize("form", ["coalesced", "per-micro-batch", "inference"])
def test_ksplit_matches_the_fp64_oracle(form, k, mb_rows, monkeypatch):
    import shallowspeed_b200.parallel.engine as engine_mod

    seen = []

    class Recording(engine_mod.Trainer):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            seen.append((self.engine.chain_cluster(), self.engine.chain_ksplit()))

    monkeypatch.setattr(engine_mod, "Trainer", Recording)
    if form == "inference":
        from shallowspeed_b200.pipe import InferenceSchedule

        eng = _trainer(_sizes(k), mb_rows, 2).worker.engine_for(InferenceSchedule(2, 1, 0))
        assert (eng.chain_cluster(), eng.chain_ksplit()) == (4, 2)
        _run(_sizes(k), mb_rows, 2, "fp32", expect_chain=True, inference=True)
    else:
        env = ("SSB_NO_COALESCE",) if form == "per-micro-batch" else ()
        _run(_sizes(k), mb_rows, 2, "fp32", expect_chain=True, env=env, monkeypatch=monkeypatch)
        # the per-micro-batch backward-only launches have no layer 1 to split, the forward launches do
        assert seen == [(4, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("k,mb_rows", [(129, 24), (200, 100)])
def test_ksplit_cross_entropy_matches_the_fp64_oracle(k, mb_rows, precision):
    from test_gpu_cross_entropy import _run_ce

    _run_ce(_sizes(k), mb_rows, 2, precision, expect_chain=True, cluster=4)


@pytest.mark.gpu
@pytest.mark.parametrize("precision,loss", [("fp32", "mse"), ("tf32", "cross_entropy")])
@pytest.mark.parametrize("k,gbs,n_mu", [(160, 128, 4), (200, 80, 2)])
def test_ksplit_dropout_matches_fp64(k, gbs, n_mu, precision, loss):
    from shallowspeed_b200.parallel.engine import Trainer
    from test_gpu_chain import check_layers
    from test_gpu_dropout import P, SEED, _batch

    sizes = _sizes(k)
    lr = 0.05
    tr = Trainer(sizes, global_batch_size=gbs, n_mubatches=n_mu, lr=lr, precision=precision, loss=loss, dropout=P,
                 dropout_seed=SEED, device="cuda:0")
    eng, model = tr.engine, tr.model
    assert eng.uses_chain() and eng.coalesced() and (eng.chain_cluster(), eng.chain_ksplit()) == (4, 2)
    W0 = model.arena.weights.detach().clone()
    x, y = _batch(gbs, sizes[0], sizes[-1], seed=3)
    tr.step(x, y)
    tr.synchronize()
    mb = gbs // n_mu
    check_layers(eng, model, W0, x, n_mu, mb, precision, lr, lambda mu: mu * mb + torch.arange(mb))
