"""Numerics of every hand-written sm_90a kernel against a plain PyTorch fp32 reference
of the same op.  TF32 tensor-core math (10-bit mantissa products, fp32 accumulate) =>
tolerances are relative to the magnitude of the result."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _K():
    from shallowspeed_b200.ops import cuda as K

    return K


def rel_err(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


SHAPES = [  # rows, in, out
    (32, 784, 128), (32, 128, 127), (32, 127, 126), (32, 126, 125), (32, 123, 10), (4, 784, 128),
    (8, 125, 124), (128, 784, 128), (16, 512, 384), (300, 200, 130), (1, 40, 7),
]


TOL = {"tf32": 3e-3, "fp32": 2e-5}     # single-pass TF32 (truncated operands) vs 3xTF32 (fp32-equivalent)


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("rows,k,n", SHAPES)
@pytest.mark.parametrize("relu", [False, True])
def test_linear_fwd(rows, k, n, relu, precision):
    K = _K()
    torch.manual_seed(rows * 7 + k + n)
    x = torch.randn(rows, k, device="cuda")
    W = torch.randn(n, k, device="cuda") / k ** 0.5
    b = torch.randn(1, n, device="cuda")
    y = K.linear_fwd(x, W, b, relu=relu, precision=precision)
    ref = x.double() @ W.double().T + b.double()
    if relu:
        ref = ref.clamp_min(0)
    assert y.shape == (rows, n)
    assert rel_err(y.double(), ref) < TOL[precision]


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("rows,k,n", SHAPES)
def test_linear_dgrad(rows, k, n, precision):
    K = _K()
    torch.manual_seed(rows + k * 3 + n)
    dz = torch.randn(rows, n, device="cuda")
    W = torch.randn(n, k, device="cuda") / n ** 0.5
    mask = torch.randn(rows, k, device="cuda")
    dx = K.linear_dgrad(dz, W, precision=precision)
    ref = dz.double() @ W.double()
    assert rel_err(dx.double(), ref) < TOL[precision]
    dxm = K.linear_dgrad(dz, W, mask=mask, precision=precision)
    assert rel_err(dxm.double(), ref * (mask > 0)) < TOL[precision]


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("rows,k,n", SHAPES)
@pytest.mark.parametrize("accumulate", [False, True])
def test_linear_wgrad(rows, k, n, accumulate, precision):
    K = _K()
    torch.manual_seed(rows + k + n * 5)
    dz = torch.randn(rows, n, device="cuda")
    x = torch.randn(rows, k, device="cuda")
    ld = (k + 1 + 7) // 8 * 8
    G = torch.randn(n, ld, device="cuda")
    G0 = G.clone()
    K.linear_wgrad(dz, x, G[:, :k], accumulate=accumulate, grad_b=G[:, k], precision=precision)
    ref_w = dz.double().T @ x.double()
    ref_b = dz.double().sum(0)
    if accumulate:
        ref_w = ref_w + G0[:, :k].double()
        ref_b = ref_b + G0[:, k].double()
    assert rel_err(G[:, :k].double(), ref_w) < TOL[precision]
    assert rel_err(G[:, k].double(), ref_b) < 1e-5      # db is an exact fp32 reduction
    pad, pad0 = G[:, k + 1:], G0[:, k + 1:]              # padding: untouched, or zeroed by the 16-byte-granular TMA store
    assert bool(((pad == pad0) | (pad == 0)).all())


def test_wgrad_fused_sgd_single_replica():
    K = _K()
    torch.manual_seed(0)
    rows, k, n, lr = 32, 128, 127, 0.05
    dz, x = torch.randn(rows, n, device="cuda"), torch.randn(rows, k, device="cuda")
    ld = 136
    W, G = torch.randn(n, ld, device="cuda"), torch.randn(n, ld, device="cuda")
    W0, G0 = W.clone(), G.clone()
    K.linear_wgrad(dz, x, G[:, :k], accumulate=False, grad_b=G[:, k], weight=W[:, :k], lr=lr, fuse_sgd=True)
    gw = dz.double().T @ x.double()
    gb = dz.double().sum(0)
    assert rel_err(W[:, :k].double(), W0[:, :k].double() - lr * gw) < 1e-3
    assert rel_err(W[:, k].double(), W0[:, k].double() - lr * gb) < 1e-5
    assert torch.equal(G, G0)


def test_loss_head_matches_reference_chain():
    from shallowspeed_b200.ops import functional as F

    K = _K()
    torch.manual_seed(1)
    for rows in (4, 32, 128):
        z = torch.randn(rows, 10, device="cuda") * 3
        t = torch.eye(10, device="cuda")[torch.randint(0, 10, (rows,), device="cuda")]
        dz, p, loss = K.loss_head_backward(z, t, 128)
        p_ref = F.softmax_ref(z.double())
        dz_ref = F.softmax_grad_ref(F.mse_loss_grad_ref(p_ref, t.double(), 128), z.double())
        assert rel_err(p.double(), p_ref) < 1e-5
        assert rel_err(dz.double(), dz_ref) < 1e-4
        assert abs(float(loss) - float(F.mse_loss_ref(p_ref, t.double(), 128))) < 1e-5
        assert rel_err(K.softmax(z).double(), p_ref) < 1e-5
        up = torch.randn(rows, 10, device="cuda")
        assert rel_err(K.softmax_grad(up, z).double(), F.softmax_grad_ref(up.double(), z.double())) < 1e-4


def test_elementwise_kernels():
    K = _K()
    torch.manual_seed(2)
    x = torch.randn(37, 123, device="cuda")
    assert torch.equal(K.relu(x), x.clamp_min(0))
    g = torch.randn(37, 123, device="cuda")
    assert torch.equal(K.relu_grad(g, x > 0), g * (x > 0))
    assert torch.equal(K.relu_grad(g, x.clamp_min(0)), g * (x > 0))
    t = torch.randn(37, 123, device="cuda")
    assert torch.allclose(K.mse_loss_grad(x, t, 128), -2 * (t - x) / 128, atol=1e-7)
    w, gr = torch.randn(100003, device="cuda"), torch.randn(100003, device="cuda")
    ref = w - 0.006 * gr
    K.sgd_step_(w, gr, 0.006)
    assert torch.allclose(w, ref, atol=1e-7)
    pred = torch.randn(128, 10, device="cuda")
    tgt = torch.eye(10, device="cuda")[torch.randint(0, 10, (128,), device="cuda")]
    assert int(K.count_correct(pred, tgt)) == int((pred.argmax(1) == tgt.argmax(1)).sum())


def test_module_path_matches_cpu():
    """The Module-level model (Linear.forward/backward on CUDA tensors -> our kernels)
    reproduces the CPU oracle within TF32 tolerance."""
    from shallowspeed_b200.layers import MLP

    sizes = [784, 128, 127, 126, 125, 124, 123, 10]
    torch.manual_seed(3)
    x = torch.randn(32, 784)
    t = torch.eye(10)[torch.randint(0, 10, (32,))]
    cpu, gpu = MLP(sizes, 0, 1, 128), MLP(sizes, 0, 1, 128).to("cuda")
    out_c = cpu.forward(x, 0)
    out_g = gpu.forward(x.cuda(), 0)
    assert rel_err(out_g.cpu(), out_c) < 5e-5
    cpu.backward(t, 0)
    gpu.backward(t.cuda(), 0)
    for pc, pg in zip(cpu.parameters(), gpu.parameters()):
        # default precision is fp32 (3xTF32): 14 chained GEMMs agree with the CPU oracle to ~1e-5 in norm
        assert float((pg.grad.cpu() - pc.grad).norm() / pc.grad.norm()) < 2e-4


# ---------------------------------------------------------------------------------------------------------
# How close to fp32 is the 3xTF32 scheme REALLY?  Same inputs through (a) our tensor-core kernels in fp32 mode and
# (b) torch.matmul in true fp32 (TF32 disabled), both measured against an fp64 oracle.  What limits 3xTF32 is not the
# operand split (error 2^-21 per product) but the tensor core's accumulate step, whose error grows with the number of
# accumulate steps, where cuBLAS' FFMA chain rounds to nearest.  The kernels therefore sum each 32-wide k-block in a fresh
# tensor-core accumulator and add the k-block sums in fp32 (ptx.cuh warp_mma_kblock).  Asserted: within 8x of cuBLAS fp32
# for K <= 2048, within 32x at K = 8192; the measured numbers are printed (-s).
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,k,n", [(32, 784, 128), (128, 784, 128), (32, 128, 127), (32, 123, 10), (128, 2048, 512), (8, 8192, 256)])
def test_3xtf32_error_next_to_cublas_fp32(rows, k, n):
    K = _K()
    torch.manual_seed(1234 + rows + k + n)
    x = torch.randn(rows, k, device="cuda")
    W = torch.randn(n, k, device="cuda") / k ** 0.5
    dz = torch.randn(rows, n, device="cuda")
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        cases = {
            "fwd": (K.linear_fwd(x, W, None, relu=False, precision="fp32")[:, :n], x @ W.T, x.double() @ W.double().T),
            "dgrad": (K.linear_dgrad(dz, W, precision="fp32")[:, :k], dz @ W, dz.double() @ W.double()),
        }
        ld = (k + 1 + 7) // 8 * 8
        G = torch.zeros(n, ld, device="cuda")
        K.linear_wgrad(dz, x, G[:, :k], accumulate=False, grad_b=G[:, k], precision="fp32")
        cases["wgrad"] = (G[:, :k], dz.T @ x, dz.double().T @ x.double())
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    for name, (ours, cublas, ref) in cases.items():
        scale = float(ref.abs().max())
        e_ours = float((ours.double() - ref).abs().max()) / scale
        e_cublas = float((cublas.double() - ref).abs().max()) / scale
        print(f"3xTF32 vs cuBLAS fp32 [{name} rows={rows} k={k} n={n}]: ours {e_ours:.3e}  cublas {e_cublas:.3e}  ratio {e_ours / max(e_cublas, 1e-12):.2f}")
        assert e_ours <= (8.0 if k <= 2048 else 32.0) * e_cublas + 2e-7, (name, e_ours, e_cublas)
