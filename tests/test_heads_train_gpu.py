"""GPU tests of the training keypoint heads (centerpose_b200.heads_train, csrc/heads_train.cu) against torch autograd
in float64 (tests/heads_train_cases.restated), in both precisions.

Accuracy: for each output and each gradient, max|dev - f64| / max|f64| and the relative L2 error must be at most
max(4 * e32, 1e-6), e32 being the same statistic of torch's fp32 autograd with cuDNN's TF32 off: the training DCN's
bound (tests/dcn_train_cases.py).
"""
import contextlib

import pytest
import torch

from centerpose_b200 import heads_train
from tests import heads_train_cases as hc
from tests.dcn_train_cases import bound_failures, stats

pytestmark = pytest.mark.gpu

DEV = hc.DEV


@contextlib.contextmanager
def _fp32_cudnn():
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        yield


def _restated(x, params, gos, dtype, need_x=True):
    with _fp32_cudnn():
        return hc.restated(x, params, gos, dtype, need_x)


@pytest.mark.parametrize("precision", hc.PRECISIONS)
@pytest.mark.parametrize("shape", hc.EXACT, ids=hc.shape_id)
def test_exact_on_integer_data(shape, precision):
    """Integer x and grad_output, dyadic weights: every sum is exact, so every output and gradient equals float64."""
    x, params, gos = hc.make_inputs(*shape, seed=sum(shape), integer=True)
    want = hc.flat(_restated(x, params, gos, torch.float64))
    got = hc.flat(hc.device(x, params, gos, precision))
    assert [n for n, _ in got] == [n for n, _ in want]
    bad = [n for (n, g), (_, w) in zip(got, want) if not torch.equal(g.double(), w)]
    assert not bad, bad


@pytest.mark.parametrize("precision", hc.PRECISIONS)
@pytest.mark.parametrize("shape", hc.ACCURACY, ids=hc.shape_id)
def test_accuracy(shape, precision):
    x, params, gos = hc.make_inputs(*shape, seed=7 * sum(shape))
    ref64 = hc.flat(_restated(x, params, gos, torch.float64))
    ref32 = hc.flat(_restated(x, params, gos, torch.float32))
    got = hc.flat(hc.device(x, params, gos, precision))
    bad = []
    for (name, g), (_, r), (_, r32) in zip(got, ref64, ref32):
        assert g.shape == r.shape and g.dtype == torch.float32 and torch.isfinite(g).all(), name
        bad += bound_failures("%s %s" % (hc.shape_id(shape), name), g, r, r32)
    worst = max(stats(g, r)[1] for (_, g), (_, r) in zip(got, ref64))
    print("%s %s: worst relative L2 %.3g" % (hc.shape_id(shape), precision, worst))
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("precision", hc.PRECISIONS)
@pytest.mark.parametrize("gated", [(1,), (0, 4), (1, 2, 3, 5), (0, 1, 2, 3, 4, 5)],
                         ids=lambda g: "none_" + "_".join(map(str, g)))
def test_gated_heads(gated, precision):
    """grad_output None for the heads in ``gated``: their parameter grads are None through autograd, and dx is the
    float64 dx of the remaining heads."""
    shape = (2, 24, 20, 18, 40)
    x, params, gos = hc.make_inputs(*shape, seed=31, integer=True)
    gos = [None if h in gated else g for h, g in enumerate(gos)]
    _, gx64, pg64 = _restated(x, params, gos, torch.float64)
    xl = x.clone().requires_grad_(True)
    leaves = [p.clone().requires_grad_(True) for p in params]
    outs = heads_train._Heads.apply(precision, xl, *leaves)
    live = [(o, g) for o, g in zip(outs, gos) if g is not None]
    if live:
        torch.autograd.backward([o for o, _ in live], [g for _, g in live])
        assert torch.equal(xl.grad.double(), gx64)
    else:
        assert xl.grad is None
    for i, (l, r) in enumerate(zip(leaves, pg64)):
        if i // 4 in gated:
            assert l.grad is None, i
        else:
            assert torch.equal(l.grad.double(), r), i


@pytest.mark.parametrize("precision", hc.PRECISIONS)
def test_x_without_grad_skips_the_data_pass(precision):
    shape = (2, 24, 20, 18, 40)
    x, params, gos = hc.make_inputs(*shape, seed=32, integer=True)
    leaves = [p.clone().requires_grad_(True) for p in params]
    outs = heads_train._Heads.apply(precision, x, *leaves)
    torch.autograd.backward(outs, gos)
    assert x.grad is None
    _, gx, grads = hc.device(x, params, gos, precision, need_x=False)
    assert gx is None
    for l, g in zip(leaves, grads):
        assert torch.equal(l.grad, g)


@pytest.mark.parametrize("precision", hc.PRECISIONS)
@pytest.mark.parametrize("shape", hc.DETERMINISM, ids=hc.shape_id)
def test_deterministic(shape, precision):
    x, params, gos = hc.make_inputs(*shape, seed=3)
    a = hc.flat(hc.device(x, params, gos, precision))
    b = hc.flat(hc.device(x, params, gos, precision))
    bad = [n for (n, u), (_, v) in zip(a, b) if not torch.equal(u, v)]
    assert not bad, bad


@pytest.mark.parametrize("precision", hc.PRECISIONS)
def test_gradients_scale_exactly(precision):
    shape = (2, 64, 40, 36, 256)
    x, params, gos = hc.make_inputs(*shape, seed=5)
    _, gx0, g0 = hc.device(x, params, gos, precision)
    for k in (-30, -10, 10):
        s = 2.0 ** k
        _, gx, g = hc.device(x, params, [t * s for t in gos], precision)
        assert torch.equal(gx, gx0 * s), "grad_x * 2^%d" % k
        for i, (a, b) in enumerate(zip(g, g0)):
            assert torch.equal(a, b * s), "parameter %d * 2^%d" % (i, k)


def test_memory():
    """DLA-34's heads at B = 8 on 128x128 maps: what stays allocated after the forward is the six outputs, within the
    allocator's 1 MiB of small-block slack (torch's autograd would keep 6 * hc * R^2 * B * 4 = 768 MiB of hidden maps
    on top); the backward's peak rise is the gradients plus at most the workspace and the per-call weight copies."""
    from centerpose_b200 import _lib
    B, C, H, W, hcn = hc.MEMORY
    torch.manual_seed(0)
    m = heads_train.KeypointHead(C, hcn).to(DEV)
    x = torch.randn(B, C, H, W, device=DEV).relu_().requires_grad_(True)
    gos = None
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    outs = m(x)
    torch.cuda.synchronize()
    kept = torch.cuda.memory_allocated(DEV) - base
    out_bytes = sum(o.numel() * 4 for o in outs)
    hidden = 6 * hcn * H * W * B * 4
    print("kept after forward %d bytes, outputs %d; the reference module keeps %d more" % (kept, out_bytes, hidden))
    assert out_bytes <= kept <= out_bytes + (1 << 20)
    gos = [torch.randn_like(o) for o in outs]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    start = torch.cuda.memory_allocated(DEV)
    torch.autograd.backward(outs, gos)
    torch.cuda.synchronize()
    grads = x.numel() * 4 + sum(p.numel() * 4 for p in m.parameters())
    ws = _lib.lib().cpb200_heads_train_workspace_bytes(B, C, H, W, hcn)
    concat = sum(p.numel() * 4 for p in m.parameters())        # the per-call concatenated weights and their grads
    rise = torch.cuda.max_memory_allocated(DEV) - start
    print("backward peak rise %d bytes: gradients %d, workspace %d" % (rise, grads, ws))
    assert rise <= grads + ws + 2 * concat + (1 << 20)


def test_training_matches_float64():
    """Five Adam steps of the heads alone on a fixed feature map, with heads_train.KeypointHead, with torch's heads in
    fp32 and in float64, from the same init: each parameter tensor within 1e-4 of its largest value of float64, or 4
    times the fp32 arm's own difference where that is larger (the training DCN's rule)."""
    torch.manual_seed(0)
    C, hcn = 32, 64
    mine = heads_train.KeypointHead(C, hcn).to(DEV)
    arms = [mine, heads_train.KeypointHead(C, hcn), heads_train.KeypointHead(C, hcn)]
    for m in arms[1:]:
        m.load_state_dict(mine.state_dict())
    dts = (torch.float32, torch.float32, torch.float64)
    arms = [arms[0]] + [m.to(DEV).to(dt) for m, dt in zip(arms[1:], dts[1:])]
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, C, 32, 32, generator=g).relu().to(DEV)
    target = [torch.randn(2, c, 32, 32, generator=g).to(DEV) for c in heads_train.OUTPUTS]
    opts = [torch.optim.Adam(m.parameters(), lr=1e-3) for m in arms]
    with _fp32_cudnn():
        for _ in range(5):
            for i, (m, opt, dt) in enumerate(zip(arms, opts, dts)):
                opt.zero_grad()
                outs = m(x.to(dt)) if i == 0 else hc.heads_torch(x.to(dt), m.head_parameters())
                loss = sum(((o - t.to(dt)) ** 2).mean() for o, t in zip(outs, target))
                loss.backward()
                opt.step()
    names = [n for n, _ in mine.named_parameters()]
    bad = []
    for name, a, b, r in zip(names, *([p.detach().double() for p in m.parameters()] for m in arms)):
        scale = r.abs().max().item()
        err, err32 = (a - r).abs().max().item() / scale, (b - r).abs().max().item() / scale
        if err > max(4 * err32, 1e-4):
            bad.append("%s: %.3g > max(4 * %.3g, 1e-4)" % (name, err, err32))
    assert not bad, "\n".join(bad)


# ---- networks ------------------------------------------------------------------------------------------------------
NET_ARCHS = ("dla_34", "res_50")


def _net_arm(arch, sd, cfg, batch, dtype, heads_fn, pins, record):
    """(loss, {parameter: gradient}) of the oracle backbone, ``heads_fn`` and train_loss_ref.loss_torch, its DCNs
    restated and pinned as in tests/test_dcn_train_models_gpu.py."""
    from oracle import dla_ref, resnet_ref, train_loss_ref
    from tests import test_dcn_train_models_gpu as dm
    leaves = {k: v.to(DEV, dtype).requires_grad_(not k.endswith(dm.NOT_DIFFERENTIATED)) for k, v in sd.items()}
    b = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
    fwd = dm.dcn_arm(pins, dm.restated_conv, [] if record else None,
                     {id(v): k[:-len(".weight")] for k, v in leaves.items()})
    backbone = dla_ref.dla34_backbone if arch == "dla_34" else resnet_ref.resnet50_backbone
    with _fp32_cudnn(), dm._dcn_module_forward(fwd):
        heads = heads_fn(leaves, backbone(leaves, b["input"]))
        loss, _ = train_loss_ref.loss_torch(heads, b, cfg.LOSS)
        params = [k for k, v in leaves.items() if v.requires_grad]
        grads = torch.autograd.grad(loss, [leaves[k] for k in params], allow_unused=True)
    return loss.detach(), {k: g for k, g in zip(params, grads) if g is not None}


def _device_heads(precision):
    def fn(leaves, feat):
        ps = [leaves["head_model.%s.%d.%s" % (h, i, n)] for h in heads_train.HEADS for i in (0, 2)
              for n in ("weight", "bias")]
        return list(heads_train._Heads.apply(precision, feat, *ps))
    return fn


@pytest.fixture(scope="module")
def net_batch(tmp_path_factory):
    from tests.train_cases import seeded_jpeg_batch
    return seeded_jpeg_batch(tmp_path_factory.mktemp("heads_models"), B=4, res=256)


@pytest.mark.parametrize("arch", NET_ARCHS)
def test_network_gradients(net_batch, arch):
    """DLA-34 (hc 256) and ResNet-50 (hc 64) on a seeded TrainData batch: the loss and every parameter's gradient of
    the device heads, in each precision, within the bound of the float64 arm; torch's fp32 heads give e32."""
    from oracle import dla_ref
    from tests import test_dcn_train_models_gpu as dm
    cfg, batch = net_batch
    sd = dm.weights(arch)
    pins = []
    loss_c, grad_c = _net_arm(arch, sd, cfg, batch, torch.float64, dla_ref.keypoint_head, pins, True)
    loss_b, grad_b = _net_arm(arch, sd, cfg, batch, torch.float32, dla_ref.keypoint_head, pins, False)
    assert any(k.startswith("head_model.") for k in grad_c)
    for precision in hc.PRECISIONS:
        loss_a, grad_a = _net_arm(arch, sd, cfg, batch, torch.float32, _device_heads(precision), pins, False)
        assert set(grad_a) == set(grad_b) == set(grad_c)
        bad = bound_failures("%s %s loss" % (arch, precision), loss_a, loss_c, loss_b)
        for k, r in grad_c.items():
            assert torch.isfinite(grad_a[k]).all(), k
            bad += bound_failures("%s %s %s" % (arch, precision, k), grad_a[k], r, grad_b[k])
        print("%s %s loss: %s (e32 %s)" % (arch, precision, stats(loss_a, loss_c), stats(loss_b, loss_c)))
        assert not bad, "\n".join(bad)
