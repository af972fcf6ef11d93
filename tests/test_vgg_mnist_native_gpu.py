"""VGG16_MNIST on the native kernels: ragged implicit-GEMM convs (28-, 14-, 7-, 3-wide maps), BatchNorm + ReLU + floor
max-pooling at odd sizes, and the VGG16_MNIST stage program of ``train/cnn_native.py``.

Kernel outputs are checked elementwise against fp64 references on the bf16-rounded operands, with bounds built the way
``token_oracles`` builds them: an fp32 accumulation term and the final bf16 rounding term."""
import copy

import pytest
import torch
import torch.nn.functional as TF

from token_oracles import U_32, U_BF, check

pytestmark = pytest.mark.gpu

F64 = torch.float64
GUARD = 64                                   # NaN elements after every output: a store from a padding row lands there
SIZES = [(28, 28), (14, 14), (7, 7), (3, 3), (5, 9), (28, 1)]
BATCHES = [1, 3, 31, 32, 33]


def _need():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from split_learning_b200.ops import native as N
    N.require()
    N.preload()
    return N


def _guarded(shape, dtype):
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[:n].view(*shape)


def _nchw(t):
    return t.to(F64).permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _operands(B, H, W, cin, cout, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, cin, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(cout, 3, 3, cin, device="cuda", generator=g) * (2.0 / (9 * cin)) ** 0.5).to(torch.bfloat16)
    bias = torch.randn(cout, device="cuda", generator=g) * 0.1
    return x, w, bias


# ------------------------------------------------------------------------------------------------ conv fwd / dgrad
def _conv_cases():
    cases = []
    for (H, W) in SIZES:
        for B in BATCHES:
            cases.append((H, W, B, 64, 128))
        cases.append((H, W, 3, 256, 512))
        cases.append((H, W, 2, 512, 512))
    return cases


@pytest.mark.parametrize("H,W,B,cin,cout", _conv_cases())
def test_ragged_conv_fwd_dgrad_fp64(H, W, B, cin, cout):
    N = _need()
    x, w, bias = _operands(B, H, W, cin, cout, seed=H * 1000 + W * 10 + B)
    K = 9 * cin
    wt = w.to(F64).permute(0, 3, 1, 2)                                   # [Cout, Cin, 3, 3]
    ref = _nhwc(TF.conv2d(_nchw(x), wt, bias.to(F64), padding=1))
    mag = _nhwc(TF.conv2d(_nchw(x).abs(), wt.abs(), bias.to(F64).abs(), padding=1))
    bound = U_BF * ref.abs() + (1 + U_BF) * (K + 2) * U_32 * mag
    for bn in (32, 64, 128, 256):
        if bn > cout:
            continue
        outs = []
        for _ in range(2):
            buf, y = _guarded((B, H, W, cout), torch.bfloat16)
            N.conv3x3_fwd(x, w, y, bias, tiling=(bn, 1))
            torch.cuda.synchronize()
            assert torch.isnan(buf[-GUARD:]).all(), "store past the output"
            check(y, ref, bound, f"fwd {H}x{W} B{B} bn{bn}")
            outs.append(y.clone())
        assert torch.equal(outs[0], outs[1])
    # input gradient: dy [B, H, W, Cout] through the same weights, mirrored taps
    dy = torch.randn(B, H, W, cout, device="cuda").to(torch.bfloat16)
    dref = _nhwc(TF.conv_transpose2d(_nchw(dy), wt, padding=1))
    dmag = _nhwc(TF.conv_transpose2d(_nchw(dy).abs(), wt.abs(), padding=1))
    dbound = U_BF * dref.abs() + (1 + U_BF) * (9 * cout + 2) * U_32 * dmag
    for bn in (64, 128, 256):
        if bn > cin:
            continue
        outs = []
        for _ in range(2):
            buf, dx = _guarded((B, H, W, cin), torch.bfloat16)
            N.conv3x3_dgrad(dy, w, dx, tiling=(bn, 1))
            torch.cuda.synchronize()
            assert torch.isnan(buf[-GUARD:]).all(), "store past the output"
            check(dx, dref, dbound, f"dgrad {H}x{W} B{B} bn{bn}")
            outs.append(dx.clone())
        assert torch.equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ wgrad
def _wgrad_cases():
    cases = []
    for (H, W) in SIZES:
        for B in (1, 3, 32, 33):
            cases.append((H, W, B, 64, 64))
        cases.append((H, W, 3, 128, 256))
        cases.append((H, W, 2, 512, 512))
    return cases


@pytest.mark.parametrize("H,W,B,cin,cout", _wgrad_cases())
def test_ragged_conv_wgrad_fp64(H, W, B, cin, cout):
    N = _need()
    g = torch.Generator(device="cuda").manual_seed(7 * H + W + B)
    x = torch.randn(B, H, W, cin, device="cuda", generator=g).to(torch.bfloat16)
    dy = torch.randn(B, H, W, cout, device="cuda", generator=g).to(torch.bfloat16)
    wshape = (cout, cin, 3, 3)
    ref = torch.nn.grad.conv2d_weight(_nchw(x), wshape, _nchw(dy), padding=1).permute(0, 2, 3, 1)
    mag = torch.nn.grad.conv2d_weight(_nchw(x).abs(), wshape, _nchw(dy).abs(), padding=1).permute(0, 2, 3, 1)
    K = B * H * W
    for ks in (1, 2, 0):
        bound = (K + max(ks, 1) + 2) * U_32 * mag + 1e-30
        for bn in (64, 128, 256):
            if bn > cin:
                continue
            outs = []
            for _ in range(2):
                dw = torch.zeros(cout, 3, 3, cin, device="cuda")
                N.conv3x3_wgrad(x, dy, dw, k_split=ks, block_n=bn)
                torch.cuda.synchronize()
                check(dw, ref, bound, f"wgrad {H}x{W} B{B} ks{ks} bn{bn}")
                outs.append(dw)
            assert torch.equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ the padded-box rule
def test_padded_box_reproduces_power_of_two_boxes():
    N = _need()
    for T in (128, 64, 32):
        for H in (32, 16, 8, 4, 2, 1):
            for W in (32, 16, 8, 4, 2, 1):
                if W > T:
                    continue
                tb, th, tw, rag = N.conv_pixel_box(H, W, T)
                assert rag == 0, (H, W, T)
                assert N.conv_pixel_box(H, W, T, padded=True)[:3] == (tb, th, tw), (H, W, T)
    # the VGG16_MNIST maps (conv / dgrad tile of 128 pixels, bf16 wgrad K step of 64)
    assert N.conv_pixel_box(28, 28, 128) == (1, 4, 32, 1)
    assert N.conv_pixel_box(14, 14, 128) == (1, 8, 16, 1)
    assert N.conv_pixel_box(7, 7, 128) == (2, 8, 8, 1)
    assert N.conv_pixel_box(3, 3, 128) == (8, 4, 4, 1)
    assert N.conv_pixel_box(28, 28, 64) == (1, 2, 32, 1)
    assert N.conv_pixel_box(14, 14, 64) == (1, 4, 16, 1)
    assert N.conv_pixel_box(7, 7, 64) == (1, 8, 8, 1)
    assert N.conv_pixel_box(3, 3, 64) == (4, 4, 4, 1)
    assert N.conv_pixel_box(2, 130, 128)[3] == -1


# ------------------------------------------------------------------------------------------------ BN + ReLU + pool
def _bn_ref(y, gamma, beta, dout, relu, eps=1e-5):
    """fp64 train-mode batch_norm -> relu -> max_pool2d (floor) on y [B, H, W, C]; (out, dy, dgamma, dbeta, mean, var)."""
    yc = _nchw(y).detach().requires_grad_(True)
    g = gamma.to(F64).detach().requires_grad_(True)
    b = beta.to(F64).detach().requires_grad_(True)
    z = TF.batch_norm(yc, None, None, g, b, True, 0.0, eps)
    a = torch.relu(z) if relu else z
    o = TF.max_pool2d(a, 2)
    o.backward(_nchw(dout))
    mean = yc.detach().mean((0, 2, 3))
    var = yc.detach().var((0, 2, 3), unbiased=False)
    xh = (yc.detach() - mean[None, :, None, None]) / torch.sqrt(var[None, :, None, None] + eps)
    return _nhwc(o.detach()), _nhwc(yc.grad), g.grad, b.grad, mean, var, _nhwc(xh)


def _bn_case(N, B, H, W, C, relu, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = (torch.randn(B, H, W, C, device="cuda", generator=g) * 1.5 + 0.3).to(torch.bfloat16)
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g) * 0.2
    rm, rv = torch.randn(C, device="cuda", generator=g) * 0.1, torch.rand(C, device="cuda", generator=g) + 0.5
    rm0, rv0 = rm.clone(), rv.clone()
    nbt = torch.zeros((), dtype=torch.long, device="cuda")
    OH, OW = H // 2, W // 2
    P = B * H * W
    stats = torch.zeros(2 * C, device="cuda")
    N.col_stats(y.view(-1, C), stats[:C], stats[C:])
    save = torch.empty(2 * C, device="cuda")
    obuf, out = _guarded((B, OH, OW, C), torch.bfloat16)
    N.bn_relu_pool_fwd(y, stats[:C], stats[C:], gamma, beta, rm, rv, nbt, save[:C], save[C:], out, H, W, relu, True)
    dout = torch.randn(B, OH, OW, C, device="cuda", generator=g).to(torch.bfloat16)
    ref, dref, dgref, dbref, mean, var, xh = _bn_ref(y, gamma, beta, dout, relu)
    torch.cuda.synchronize()
    what = f"{B}x{H}x{W} relu={relu}"
    assert torch.isnan(obuf[-GUARD:]).all()
    depth = P / 32 + 8                                   # fp32 statistic sums: reduction depth of the column sums
    e_xh = depth * U_32 * (1 + xh * xh)
    e_a = gamma.to(F64).abs() * e_xh + 2.0 ** -22 * (xh * gamma.to(F64)).abs() + U_32 * beta.to(F64).abs()
    e_out = _nhwc(TF.max_pool2d(_nchw(e_a), 2))         # max is 1-Lipschitz: the window's largest term bounds it
    check(out, ref, U_BF * ref.abs() + (1 + U_BF) * e_out, "bn fwd " + what)
    # running statistics cover every pre-pool pixel; num_batches_tracked
    assert int(nbt) == 1
    assert torch.allclose(rm.double(), 0.9 * rm0.double() + 0.1 * mean, rtol=1e-5, atol=1e-5)
    assert torch.allclose(rv.double(), 0.9 * rv0.double() + 0.1 * var * P / (P - 1), rtol=1e-4, atol=1e-5)
    dg = torch.zeros(C, device="cuda")
    db = torch.zeros(C, device="cuda")
    dbuf, dy = _guarded((B, H, W, C), torch.bfloat16)
    N.bn_relu_pool_bwd(dout, y, gamma, beta, save[:C], save[C:], dg, db, dy, H, W, relu, True)
    torch.cuda.synchronize()
    assert torch.isnan(dbuf[-GUARD:]).all()
    assert not torch.isnan(dy).any(), "a pre-pool pixel got no gradient"
    # |dz| upper bound on the pre-pool grid: every pixel of a window may take the window's gradient
    dzf = torch.zeros(B, H, W, C, dtype=F64, device="cuda")
    dzf[:, :2 * OH, :2 * OW] = _nhwc(TF.interpolate(_nchw(dout).abs(), scale_factor=2, mode="nearest"))
    sc = (gamma.to(F64) / torch.sqrt(var + 1e-5)).abs()
    e_k1 = depth * U_32 * dzf.mean((0, 1, 2))
    e_k2 = depth * U_32 * (dzf * xh.abs()).mean((0, 1, 2)) + (dzf * e_xh).mean((0, 1, 2))
    k2 = dgref.abs() / P
    e_dy = sc * (e_k1 + xh.abs() * e_k2 + k2 * e_xh) + depth * U_32 * dref.abs() + 2.0 ** -22 * sc * dzf
    check(dy, dref, U_BF * dref.abs() + (1 + U_BF) * e_dy, "bn bwd " + what)
    # the dropped last row / column: no pooled gradient, but the BatchNorm mean terms reach it
    if H % 2:
        check(dy[:, H - 1], dref[:, H - 1], (U_BF * dref.abs() + (1 + U_BF) * e_dy)[:, H - 1], "dropped row")
        assert dy[:, H - 1].abs().sum() > 0
    if W % 2:
        assert dy[:, :, W - 1].abs().sum() > 0
    e_dg = depth * U_32 * (dzf * xh.abs()).sum((0, 1, 2)) + (dzf * e_xh).sum((0, 1, 2))
    check(dg, dgref, e_dg + 1e-30, "dgamma " + what)
    check(db, dbref, depth * U_32 * dzf.sum((0, 1, 2)) + 1e-30, "dbeta " + what)


@pytest.mark.parametrize("H,W", [(7, 7), (3, 3), (5, 5), (28, 28)])
@pytest.mark.parametrize("relu", [True, False])
def test_bn_relu_pool_odd_fp64(H, W, relu):
    """Batch 32 (the channel-owned backward for the small maps) and a batch whose map count exceeds
    BN_BWD_CHAN_MAX_P pixels (the two-pass reduce / apply backward)."""
    N = _need()
    for B in (32, N.BN_BWD_CHAN_MAX_P // (H * W) + 1):
        _bn_case(N, B, H, W, 64, relu, seed=H * 3 + int(relu) + B)


# ------------------------------------------------------------------------------------------------ host checks
def test_ragged_host_checks():
    N = _need()
    B, H, W, C = 2, 7, 7, 64
    x, w, bias = _operands(B, H, W, C, C, seed=1)
    y = torch.empty(B, H, W, C, dtype=torch.bfloat16, device="cuda")
    acc = torch.zeros(4 * B * H * W * C, device="cuda")
    ctr = torch.zeros(64, dtype=torch.int32, device="cuda")
    s1, s2 = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    before = N.LAUNCHES
    with pytest.raises(N.NativeError, match="-14"):
        N.conv3x3_fwd(x, w, y, bias, acc=acc, tiling=(64, 2), counters=ctr)          # split-K
    with pytest.raises(N.NativeError, match="-14"):
        N.conv3x3_fwd(x, w, y, bias, col_sum=s1, col_sumsq=s2, tiling=(64, 1))      # BN statistics
    with pytest.raises(N.NativeError, match="-14"):
        N.conv3x3_dgrad(x, w, y, tiling=(64, 1), bn_stats=(y, s1, s2, s1, s2, True, False, s1, s2))
    tk = torch.zeros(4, dtype=torch.int32, device="cuda")
    with pytest.raises(N.NativeError, match="-14"):
        N.conv3x3_dgrad(x, w, y, tiling=(64, 1), publish=(tk, tk[1:].data_ptr(), tk[2:]))
    xw = torch.zeros(1, 2, 130, C, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(N.NativeError, match="-11"):
        N.conv3x3_fwd(xw, w, torch.empty(1, 2, 130, C, dtype=torch.bfloat16, device="cuda"), tiling=(64, 1))
    with pytest.raises(N.NativeError, match="-11"):
        N.conv3x3_wgrad(xw, xw, torch.zeros(C, 3, 3, C, device="cuda"))
    # BN: the grid-barrier backward and the inference forward pool even maps only
    g, b = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    out = torch.empty(B, 3, 3, C, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(N.NativeError, match="-2"):
        N.bn_relu_pool_infer(y, g, b, s1, g, out, H, W, True, True)
    bar = torch.zeros(4, dtype=torch.int32, device="cuda")
    with pytest.raises(N.NativeError, match="-2"):
        N.bn_relu_pool_bwd(out, y, g, b, s1, g, s1, s2, torch.empty_like(y), H, W, True, True, grid_bar=bar)
    assert N.LAUNCHES == before
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ stages and API
def _cos(a, b):
    a, b = a.float().flatten(), b.float().flatten()
    return (a @ b / (a.norm() * b.norm() + 1e-12)).item()


@pytest.mark.parametrize("start,end", [(0, 7), (7, 14), (14, 24), (24, 34), (34, 44), (44, 51)])
def test_vgg_mnist_shallow_stage_matches_torch(start, end):
    """Stem, ragged convs at 28 / 14 / 7 / 3, convs at 1x1, BN + ReLU + pool (even and odd), flatten, Linear + ReLU.
    Dropout is set to p = 0 on both sides (its masks are not the torch masks)."""
    _need()
    from split_learning_b200.models import VGG16_MNIST
    from split_learning_b200.train.cnn_native import nativize
    torch.manual_seed(0)
    ref = VGG16_MNIST(start, end).cuda().train()
    for mod in ref.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    nat = nativize(copy.deepcopy(ref))
    x = VGG16_MNIST.example_input(32, device="cuda")
    if start:
        with torch.no_grad():
            x = VGG16_MNIST(0, start).cuda().train()(x)
    xr = x.clone().requires_grad_(start > 0)
    xn = x.clone().requires_grad_(start > 0)
    yr = ref(xr)
    yn = nat(xn).float()
    assert yn.shape == yr.shape
    assert _cos(yn, yr) > 0.998, _cos(yn, yr)
    gr = torch.randn_like(yr)
    yr.backward(gr)
    yn.backward(gr)
    if start:
        assert _cos(xn.grad, xr.grad) > 0.98, ("dx", _cos(xn.grad, xr.grad))
    bad = []
    refp = dict(ref.named_parameters())
    for (k, pr), (_, pn) in zip(ref.named_parameters(), nat.named_parameters()):
        wk = k.replace(".bias", ".weight")
        if k.endswith(".bias") and wk in refp and refp[wk].dim() == 4 and pr.grad.norm() < 1e-3 * refp[wk].grad.norm():
            continue                                   # conv bias under train-mode BN: exactly zero gradient (noise)
        c = _cos(pn.grad, pr.grad)
        if c < 0.97:
            bad.append((k, round(c, 4)))
    assert not bad, bad
    for (k, br), (_, bn) in zip(ref.named_buffers(), nat.named_buffers()):
        if "num_batches" in k:
            assert int(br) == int(bn) == 1
        else:
            assert torch.allclose(br, bn, rtol=3e-2, atol=3e-3), k


def test_vgg_mnist_trains_through_executor():
    """Two VGG16_MNIST stages cut at 7 through make_executor: native, graph-captured, the loss falls, and the state-dict
    is the stock model's."""
    _need()
    from split_learning_b200.models import VGG16_MNIST
    from split_learning_b200.train.executor import TorchExecutor, make_executor
    learning = {"learning-rate": 0.01, "momentum": 0.5}
    torch.manual_seed(3)
    e1 = make_executor(VGG16_MNIST(0, 7), "VGG16", learning, "cuda", True, False)
    e2 = make_executor(VGG16_MNIST(7, 51), "VGG16", learning, "cuda", False, True)
    assert isinstance(e1, TorchExecutor) and isinstance(e2, TorchExecutor)
    assert e1.native and e2.native and e1.graphs and e2.graphs
    g = torch.Generator().manual_seed(5)
    x = torch.randn(32, 1, 28, 28, generator=g)
    y = torch.randint(0, 10, (32,), generator=g)
    losses = []
    for it in range(40):
        a = e1.forward_only(it, x)
        gx = e2.forward_backward_last(a, y)
        e1.backward(it, gx)
        losses.append(e2.last_loss())
    assert all(l == l for l in losses)
    assert sum(losses[-5:]) < 0.6 * sum(losses[:5]), losses[::5]
    for ex, (s, e) in ((e1, (0, 7)), (e2, (7, 51))):
        sd = ex.state_dict()
        stock = VGG16_MNIST(s, e)
        assert list(sd.keys()) == list(stock.state_dict().keys())
        assert all(torch.isfinite(v.float()).all() for v in sd.values())
        stock.load_state_dict({k: v.cpu() for k, v in sd.items()})


def test_vgg_mnist_public_api_host_plane(tmp_path):
    """One Vanilla_SL round of VGG16 / MNIST on the host plane through the native executor, with gradient clipping."""
    _need()
    from split_learning_b200.checkpoint import load_checkpoint
    from split_learning_b200.config import normalize
    from split_learning_b200.runner import run_variant
    raw = {"server": {"global-round": 1, "clients": [1, 1], "no-cluster": {"cut-layers": [7]}, "model": "VGG16",
                      "data-name": "MNIST", "parameters": {"load": False, "save": True}, "validation": False,
                      "data-distribution": {"non-iid": False, "num-sample": 128, "num-label": 10, "dirichlet": {"alpha": 1}},
                      "random-seed": 1},
           "log_path": str(tmp_path), "debug_mode": False,
           "learning": {"learning-rate": 0.01, "momentum": 0.5, "batch-size": 32, "control-count": 2, "clip-grad-norm": 1.0},
           "b200": {"algorithm": "vanilla_sl", "synthetic-data": True, "watchdog-seconds": 120}}
    srv = run_variant(normalize(raw), [dict(layer_id=1), dict(layer_id=2)], workdir=str(tmp_path), devices=["cuda:0"],
                      timeout=300)
    assert srv.history and srv.history[0]["ok"]
    sd = load_checkpoint(str(tmp_path / "VGG16_MNIST.pth"))
    from split_learning_b200.models import VGG16_MNIST
    assert list(sd.keys()) == list(VGG16_MNIST().state_dict().keys())
    assert len(sd) == 97 and all(torch.isfinite(v.float()).all() for v in sd.values())
