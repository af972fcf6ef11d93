"""Split-K without waiting: the sliced fp32 Linear kernels and the conv forward / input gradient store one partial per
slice, and one reader adds the slices in slice order (the kernel consuming a Linear result; the last slice of a conv tile
to arrive).  Checked against float64 references, bitwise against the same slices added in order by torch or by the
turn-ordered red.add path, bitwise from run to run and across graph replays, for the flush-to-zero rounding of
red.global.add, for self-resetting tile counters, and for the rejection of short partial buffers."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
SHAPES = [(512, 4096), (4096, 4096), (4096, 10)]          # (in, out) of the VGG16 classifier
BATCHES = [1, 31, 32, 33]


def _need():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from split_learning_b200.ops import native as N
    N.require()
    N.preload()
    return N


def _ordered_sum(parts):
    """+0 plus each slice in slice order, in fp32 round-to-nearest (no subnormals occur in these inputs)."""
    s = torch.zeros_like(parts[0])
    for z in range(parts.shape[0]):
        s = s + parts[z]
    return s


def _fp32_bound(a, b):
    """Elementwise bound on an fp32 dot product of length K against float64: K * 2^-23 * (|a| @ |b|)."""
    K = a.shape[1]
    return K * 2.0 ** -23 * (a.double().abs() @ b.double().abs()) + 1e-30


def _buffer(N, dgrad, fin, fout, B):
    n = N.linear_f32_slices(dgrad, fout, fin) * B * (fin if dgrad else fout)
    return torch.full((n,), float("nan"), device=DEV)          # every element must be stored before it is read


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("fin,fout", SHAPES)
def test_linear_fwd_partials(fin, fout, B):
    N = _need()
    g = torch.Generator(device=DEV).manual_seed(fin + fout + B)
    x = torch.randn(B, fin, device=DEV, generator=g)
    w = torch.randn(fout, fin, device=DEV, generator=g) / fin ** 0.5
    bias = torch.randn(fout, device=DEV, generator=g)
    part = _buffer(N, False, fin, fout, B)
    pv = N.linear_fwd_f32(x, w, part)
    assert pv.shape == (N.linear_f32_slices(False, fout, fin), B, fout)
    out = torch.empty(B, fout, device=DEV)
    N.linear_finalize(pv, bias, out, None, None, False)
    torch.cuda.synchronize()
    ref = x.double() @ w.double().t()
    err = (pv.double().sum(0) - ref).abs()
    assert bool((err <= _fp32_bound(x, w.t())).all()), float((err / _fp32_bound(x, w.t())).max())
    assert torch.equal(out, _ordered_sum(pv) + bias)
    again = torch.empty_like(out)
    N.linear_finalize(N.linear_fwd_f32(x, w, part), bias, again, None, None, False)
    torch.cuda.synchronize()
    assert torch.equal(out, again)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("fin,fout", SHAPES)
def test_linear_dgrad_partials(fin, fout, B):
    N = _need()
    g = torch.Generator(device=DEV).manual_seed(7 * (fin + fout) + B)
    w = torch.randn(fout, fin, device=DEV, generator=g) / fin ** 0.5
    ldz = fout if fout % 16 == 0 else 16
    dzp = torch.randn(B, ldz, device=DEV, generator=g)
    dz = dzp[:, :fout]
    part = _buffer(N, True, fin, fout, B)
    pv = N.linear_dgrad_f32(dz, w, part)
    assert pv.shape == (N.linear_f32_slices(True, fout, fin), B, fin)
    ref = dz.double() @ w.double()
    dx = torch.empty(B, fin, device=DEV)
    N.dropout_bwd(pv, None, dx, 0.0)                            # feeding a dropout / conv block / the stage input
    y = torch.randn(B, fin, device=DEV, generator=g)
    dzz, dbias = torch.empty(B, fin, device=DEV), torch.empty(fin, device=DEV)
    N.linear_bwd_prep(pv, y, None, dzz, dbias, True)            # feeding a Linear block
    torch.cuda.synchronize()
    err = (pv.double().sum(0) - ref).abs()
    assert bool((err <= _fp32_bound(dz, w)).all())
    s = _ordered_sum(pv)
    assert torch.equal(dx, s)
    assert torch.equal(dzz, torch.where(y > 0, s, torch.zeros_like(s)))
    again = torch.empty_like(dx)
    N.dropout_bwd(N.linear_dgrad_f32(dz, w, part), None, again, 0.0)
    torch.cuda.synchronize()
    assert torch.equal(dx, again)


def test_slice_sum_flushes_like_red_add():
    """red.global.add.f32 flushes subnormal operands and results and starts from +0: a lone -0 slice gives +0, a
    subnormal slice adds nothing."""
    N = _need()
    tiny = 2.0 ** -130                                          # subnormal in fp32
    parts = torch.tensor([[[-0.0, tiny, 1.0, tiny, -tiny]],
                          [[-0.0, 0.0, tiny, tiny, -0.0]]], device=DEV)
    out = torch.empty(1, 5, device=DEV)
    N.dropout_bwd(parts, None, out, 0.0)
    torch.cuda.synchronize()
    want = torch.tensor([[0.0, 0.0, 1.0, 0.0, 0.0]])
    assert torch.equal(out.cpu(), want)
    assert not torch.signbit(out.cpu()).any()


def test_partial_buffer_too_small_is_rejected():
    N = _need()
    x = torch.randn(32, 4096, device=DEV)
    w = torch.randn(4096, 4096, device=DEV)
    small = torch.empty(N.linear_f32_slices(False, 4096, 4096) * 32 * 4096 - 1, device=DEV)
    with pytest.raises(N.NativeError):
        N.linear_fwd_f32(x, w, small)
    small = torch.empty(N.linear_f32_slices(True, 4096, 4096) * 32 * 4096 - 1, device=DEV)
    with pytest.raises(N.NativeError):
        N.linear_dgrad_f32(x, w, small)


def test_flagship_slice_counts():
    """The sliced launches of the VGG16 classifier at batch 32 (their tiling is unchanged by the partial stores)."""
    N = _need()
    assert [N.linear_f32_slices(False, o, i) for i, o in SHAPES] == [4, 4, 32]
    assert [N.linear_f32_slices(True, o, i) for i, o in SHAPES[:2]] == [128, 64]


def test_linear_native_capacity_check():
    """The C entry points reject a partial buffer one float short before any launch (-3), independently of Python."""
    N = _need()
    from ctypes import c_int, c_longlong, c_void_p
    x, w = torch.randn(32, 4096, device=DEV), torch.randn(4096, 4096, device=DEV)
    need = N.linear_f32_slices(False, 4096, 4096) * 32 * 4096
    part = torch.empty(need, device=DEV)
    st = c_void_p(torch.cuda.current_stream().cuda_stream)
    args = lambda cap: (c_void_p(x.data_ptr()), c_void_p(w.data_ptr()), c_void_p(part.data_ptr()), c_longlong(cap), c_int(32),
                        c_int(4096), c_int(4096), c_int(4096), c_int(4096), st)
    assert N.lib().slb_linear_fwd_f32(*args(need - 1)) == -3
    assert N.lib().slb_linear_dgrad_f32(*args(N.linear_f32_slices(True, 4096, 4096) * 32 * 4096 - 1)) == -3
    assert N.lib().slb_linear_fwd_f32(*args(need)) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- conv split-K (tf32)
# (B, H, W, Cin, Cout, flip): the flagship's split-K layers, an M tail (B = 3 at 8x8: 192 rows) and the 2x2 dgrad
CONV = [(32, 8, 8, 128, 256, 0), (3, 8, 8, 256, 256, 0), (32, 4, 4, 256, 512, 0), (32, 2, 2, 512, 512, 0),
        (32, 8, 8, 128, 256, 1), (3, 8, 8, 256, 256, 1), (32, 2, 2, 512, 512, 1)]
KS = [2, 3, 5, 16, 0]                                          # 0: one K iteration per slice (k_split = k_iters)


def _conv_case(B, H, W, Cin, Cout, flip, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randn(Cout, 3, 3, Cin, device=DEV, generator=g) / (9 * Cin) ** 0.5
    a = torch.randn(B, H, W, Cout if flip else Cin, device=DEV, generator=g)
    return a, w


def _conv_ref(a, w, flip):
    """float64 conv3x3 (forward) or its input gradient, NHWC."""
    import torch.nn.functional as F
    wd = w.double().permute(0, 3, 1, 2)
    ad = a.double().permute(0, 3, 1, 2)
    if flip:
        ref = F.conv_transpose2d(ad, wd, padding=1)
    else:
        ref = F.conv2d(ad, wd, padding=1)
    return ref.permute(0, 2, 3, 1)


def _run_conv(N, a, w, out, flip, bn, ks, acc, ctr, bias=None, s1=None, s2=None):
    if flip:
        N.conv3x3_dgrad(a, w, out, acc=acc, tiling=(bn, ks), counters=ctr)
    else:
        N.conv3x3_fwd(a, w, out, bias, s1, s2, acc=acc, tiling=(bn, ks), counters=ctr)


@pytest.mark.parametrize("ks", KS)
@pytest.mark.parametrize("case", CONV)
def test_conv_split_k_last_arriver(case, ks):
    N = _need()
    B, H, W, Cin, Cout, flip = case
    a, w = _conv_case(B, H, W, Cin, Cout, flip, seed=sum(case) + ks)
    Nout, Ca, M = (Cin if flip else Cout), (Cout if flip else Cin), B * H * W
    k_iters = 9 * (Ca // 32)
    ks = ks or k_iters
    ref = _conv_ref(a, w, flip)
    bias = None if flip else torch.randn(Nout, device=DEV)
    if bias is not None:
        ref = ref + bias.double()
    ctr = torch.zeros(4096, device=DEV, dtype=torch.int32)
    for bn in (32, 64, 128, 256):
        if Nout % bn:
            continue
        acc = torch.full((N.conv_partial_floats(M, Nout, ks),), float("nan"), device=DEV)   # stored before read
        outs = []
        for _ in range(2):                                     # bitwise on a repeat
            y = torch.empty(B, H, W, Nout, device=DEV)
            s1, s2 = (None, None) if flip else (torch.zeros(Nout, device=DEV), torch.zeros(Nout, device=DEV))
            _run_conv(N, a, w, y, flip, bn, ks, acc, ctr, bias, s1, s2)
            outs.append((y, s1, s2))
        torch.cuda.synchronize()
        assert int(ctr.abs().sum()) == 0, "tile counters must be zero at rest"
        (y, s1, s2), (y2, t1, t2) = outs
        err = float((y.double() - ref).abs().max() / ref.abs().max())
        assert err < 4e-3, (bn, ks, err)                       # the selftest's tf32 tolerance
        assert torch.equal(y, y2)
        if not flip:
            assert torch.equal(s1, t1) and torch.equal(s2, t2)
            assert float((s1 - y.sum((0, 1, 2))).abs().max() / y.sum((0, 1, 2)).abs().max()) < 1e-3
        # the same slices added in slice order by the turn-ordered red.add path and the stand-alone finalize kernel
        zacc = torch.zeros(M * Nout, device=DEV)
        y3 = torch.empty_like(y)
        if flip:
            N.conv3x3_dgrad(a, w, y3, acc=zacc, tiling=(bn, ks))
        else:
            N.conv3x3_fwd(a, w, y3, bias, None, None, acc=zacc, tiling=(bn, ks))
        torch.cuda.synchronize()
        assert torch.equal(y, y3), (bn, ks)


def test_conv_partial_buffer_too_small_is_rejected():
    N = _need()
    a, w = _conv_case(32, 2, 2, 512, 512, 0, seed=1)
    y = torch.empty(32, 2, 2, 512, device=DEV)
    ctr = torch.zeros(4096, device=DEV, dtype=torch.int32)
    short = torch.empty(N.conv_partial_floats(128, 512, 16) - 1, device=DEV)
    with pytest.raises(N.NativeError):
        N.conv3x3_fwd(a, w, y, None, None, None, acc=short, tiling=(64, 16), counters=ctr)


def test_conv_split_k_graph_replay_and_publish():
    """Captured in a CUDA graph and replayed: same bits every replay, tile counters and the publish ticket back at zero,
    and the cut-head dgrad's mailbox flag released once per replay."""
    N = _need()
    dy, w = _conv_case(32, 2, 2, 512, 512, 1, seed=3)
    acc = torch.empty(N.conv_partial_floats(128, 512, 16), device=DEV)
    ctr = torch.zeros(4096, device=DEV, dtype=torch.int32)
    ticket, flag, seq = (torch.zeros(1, device=DEV, dtype=torch.int32) for _ in range(3))
    dx = torch.empty(32, 2, 2, 512, device=DEV)
    ref = torch.empty_like(dx)
    N.conv3x3_dgrad(dy, w, ref, acc=acc, tiling=(64, 16), counters=ctr)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        N.conv3x3_dgrad(dy, w, dx, acc=acc, tiling=(64, 16), counters=ctr, publish=(ticket, flag, seq))   # warm-up
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        N.conv3x3_dgrad(dy, w, dx, acc=acc, tiling=(64, 16), counters=ctr, publish=(ticket, flag, seq))
    for i in range(3):
        dx.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(dx, ref)
        assert int(ctr.abs().sum()) == 0 and int(ticket) == 0
        assert int(flag) == int(seq) == i + 2


@pytest.mark.parametrize("ks", [2, 5, 0])
@pytest.mark.parametrize("pool", [False, True])
def test_conv_dgrad_bn_stats_split_k(pool, ks):
    """bf16 dgrad whose epilogue also reduces the upstream block's BatchNorm backward sums, at forced k_split: dX is the
    plain split-K dgrad bit for bit, and the sums match the stand-alone BatchNorm backward."""
    N = _need()
    B, H, W, Cin, Cout = 32, 4, 4, 256, 512
    g = torch.Generator(device=DEV).manual_seed(11 + ks)
    w = (torch.randn(Cout, 3, 3, Cin, device=DEV, generator=g) / (9 * Cin) ** 0.5).to(torch.bfloat16)
    dy = torch.randn(B, H, W, Cout, device=DEV, generator=g).to(torch.bfloat16)
    uh, uw = (2 * H, 2 * W) if pool else (H, W)
    up_y = (torch.randn(B, uh, uw, Cin, device=DEV, generator=g) * 1.5 + 0.2).to(torch.bfloat16)
    mean = up_y.float().mean((0, 1, 2))
    istd = (up_y.float().var((0, 1, 2), unbiased=False) + 1e-5).rsqrt()
    gamma = torch.rand(Cin, device=DEV, generator=g) + 0.5
    beta = torch.randn(Cin, device=DEV, generator=g) * 0.3
    ks = ks or 9 * (Cout // 64)
    M = B * H * W
    acc = torch.empty(N.conv_partial_floats(M, Cin, ks), device=DEV)
    ctr = torch.zeros(4096, device=DEV, dtype=torch.int32)
    dx = torch.empty(B, H, W, Cin, device=DEV, dtype=torch.bfloat16)
    dgamma, dbeta = torch.zeros(Cin, device=DEV), torch.zeros(Cin, device=DEV)
    N.conv3x3_dgrad(dy, w, dx, acc=acc, tiling=(128, ks), counters=ctr,
                    bn_stats=(up_y, mean, istd, gamma, beta, True, pool, dgamma, dbeta))
    dx2 = torch.empty_like(dx)
    N.conv3x3_dgrad(dy, w, dx2, acc=acc, tiling=(128, ks), counters=ctr)
    g2, b2 = torch.zeros(Cin, device=DEV), torch.zeros(Cin, device=DEV)
    N.bn_relu_pool_bwd(dx2, up_y, gamma, beta, mean, istd, g2, b2, torch.empty_like(up_y), uh, uw, True, pool)
    torch.cuda.synchronize()
    assert int(ctr.abs().sum()) == 0
    assert torch.equal(dx, dx2)
    for got, want in ((dgamma, g2), (dbeta, b2)):
        assert float((got - want).abs().max() / want.abs().max()) < 1.5e-2      # the selftest's bf16 tolerance
