"""Token-model kernels (ops/csrc/transformer.cu + wgmma GEMM epilogues) against plain PyTorch fp32 references,
then whole KWT / ViT / BERT stages through ``nativize`` against the stock torch modules."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


def _need():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from split_learning_b200.ops import native as N
    N.require()
    N.preload()
    return N


def _close(a, b, tol, what=""):
    a, b = a.float(), b.float()
    err = (a - b).abs().max().item()
    ref = b.abs().max().item() + 1e-6
    assert err / ref < tol, f"{what}: max err {err:.4g} vs scale {ref:.4g} (rel {err / ref:.3g} >= {tol})"


def _cos(a, b):
    a, b = a.float().flatten(), b.float().flatten()
    return (a @ b / (a.norm() * b.norm() + 1e-12)).item()


@pytest.mark.parametrize("m,k,n,act,res", [(8 * 99, 64, 192, None, False), (4 * 128, 768, 3072, "gelu", False),
                                            (4 * 128, 3072, 768, None, True), (32, 768, 768, "tanh", False),
                                            (32, 64, 10, None, False), (8 * 98, 40, 64, None, False),
                                            (300, 128, 256, "relu", True)])
def test_linear_fwd_bwd(m, k, n, act, res):
    _need()
    from split_learning_b200.ops import nn as F
    torch.manual_seed(0)
    dev = "cuda"
    x = torch.randn(m, k, device=dev).to(BF)
    w = torch.nn.Parameter(torch.randn(n, k, device=dev) / math.sqrt(k))
    b = torch.nn.Parameter(torch.randn(n, device=dev) * 0.1)
    r = torch.randn(m, n, device=dev).to(BF) if res else None
    dy = torch.randn(m, n, device=dev).to(BF)
    xn = x.clone().requires_grad_(True)
    rn = r.clone().requires_grad_(True) if res else None
    y = F.linear(xn, w, b, act, rn)
    y.backward(dy)
    gw, gb = w.grad.clone(), b.grad.clone()
    w.grad = b.grad = None
    # fp32 reference on the same bf16-rounded operands
    xr = x.float().requires_grad_(True)
    wr = w.detach().to(BF).float().requires_grad_(True)
    br = b.detach().clone().requires_grad_(True)
    rr = r.float().requires_grad_(True) if res else None
    z = xr @ wr.t() + br + (rr if res else 0)
    yr = {None: lambda t: t, "gelu": torch.nn.functional.gelu, "tanh": torch.tanh, "relu": torch.relu}[act](z)
    yr.backward(dy.float())
    _close(y, yr, 2e-2, "y")
    _close(xn.grad, xr.grad, 3e-2, "dx")
    _close(gw, wr.grad, 3e-2, "dw")
    _close(gb, br.grad, 3e-2, "db")
    if res:
        _close(rn.grad, rr.grad, 3e-2, "dres")


@pytest.mark.parametrize("rows,d,res", [(8 * 99, 64, False), (520, 128, True), (4 * 128, 768, True), (8, 64, False)])
def test_layernorm_fwd_bwd(rows, d, res):
    _need()
    from split_learning_b200.ops import nn as F
    torch.manual_seed(1)
    x = (torch.randn(rows, d, device="cuda") * 2 + 0.5).to(BF)
    r = torch.randn(rows, d, device="cuda").to(BF) if res else None
    g = torch.nn.Parameter(torch.rand(d, device="cuda") + 0.5)
    b = torch.nn.Parameter(torch.randn(d, device="cuda") * 0.1)
    dy = torch.randn(rows, d, device="cuda").to(BF)
    xn = x.clone().requires_grad_(True)
    rn = r.clone().requires_grad_(True) if res else None
    y = F.layer_norm(xn, g, b, 1e-5, rn)
    y.backward(dy)
    gg, gb = g.grad.clone(), b.grad.clone()
    xr = x.float().requires_grad_(True)
    rr = r.float().requires_grad_(True) if res else None
    gr, br = g.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
    pre = xr + rr if res else xr
    if res:
        pre = pre + (pre.detach().to(BF).float() - pre.detach())   # the kernel normalises the bf16-rounded sum
    yr = torch.nn.functional.layer_norm(pre, (d,), gr, br, 1e-5)
    yr.backward(dy.float())
    _close(y, yr, 2e-2, "y")
    _close(xn.grad, xr.grad, 3e-2, "dx")
    _close(gg, gr.grad, 3e-2, "dgamma")
    _close(gb, br.grad, 3e-2, "dbeta")
    if res:
        _close(rn.grad, rr.grad, 3e-2, "dres")


def _attn_ref(q, k, v, heads, bias=None, mask=None, p=0.0):
    b, s, e = q.shape
    dh = e // heads
    sp = lambda t: t.view(b, s, heads, dh).transpose(1, 2)
    sc = sp(q) @ sp(k).transpose(-1, -2) / math.sqrt(dh)
    if bias is not None:
        sc = sc + bias[:, None, None, :]
    pr = torch.softmax(sc, -1)
    if mask is not None:
        pr = pr * mask / (1 - p)
    return (pr @ sp(v)).transpose(1, 2).reshape(b, s, e)


@pytest.mark.parametrize("b,s,e,heads,packed,bias", [(8, 99, 64, 1, True, False), (6, 65, 128, 4, True, False),
                                                       (3, 128, 768, 12, False, True), (5, 50, 128, 4, True, False),
                                                       (2, 17, 64, 2, False, False)])
def test_attention_fwd_bwd(b, s, e, heads, packed, bias):
    _need()
    from split_learning_b200.ops import nn as F
    torch.manual_seed(2)
    dev = "cuda"
    kb = None
    if bias:
        kb = torch.zeros(b, s, device=dev)
        kb[:, s - 9:] = -10000.0
    do = torch.randn(b, s, e, device=dev).to(BF)
    if packed:
        qkv = torch.randn(b, s, 3 * e, device=dev).to(BF)
        qn = qkv.clone().requires_grad_(True)
        out = F.attention_packed(qn, heads, 0.0, kb)
        out.backward(do)
        got = qn.grad
        qr = qkv.float().requires_grad_(True)
        ref = _attn_ref(qr[..., :e], qr[..., e:2 * e], qr[..., 2 * e:], heads, kb)
        ref.backward(do.float())
        want = qr.grad
    else:
        q, k, v = (torch.randn(b, s, e, device=dev).to(BF) for _ in range(3))
        qn, kn, vn = (t.clone().requires_grad_(True) for t in (q, k, v))
        out = F.attention(qn, kn, vn, heads, (0, 0, 0), kb)
        out.backward(do)
        got = torch.cat([qn.grad, kn.grad, vn.grad], -1)
        qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
        ref = _attn_ref(qr, kr, vr, heads, kb)
        ref.backward(do.float())
        want = torch.cat([qr.grad, kr.grad, vr.grad], -1)
    _close(out, ref, 2e-2, "out")
    _close(got, want, 4e-2, "dqkv")
    assert _cos(got, want) > 0.999


def test_attention_dropout_consistent():
    """Probability dropout: recover the mask with V = I, then check forward and backward against the masked reference."""
    N = _need()
    torch.manual_seed(3)
    dev, b, s, h, dh, p, seed = "cuda", 3, 64, 2, 64, 0.25, 1234
    e = h * dh
    q, k = (torch.randn(b, s, e, device=dev).to(BF) for _ in range(2))
    eye = torch.eye(s, device=dev).to(BF).repeat(b, 1, h)                 # [b, s, h*dh] with dh == s
    out = torch.empty(b, s, e, device=dev, dtype=BF)
    lse = torch.empty(b * h * 128, device=dev)
    N.attn_fwd(q, k, eye, e, e, e, 0, 0, 0, out, e, lse, None, b, s, h, dh, p, seed)
    mask = (out.view(b, s, h, dh).transpose(1, 2) != 0).float()           # [b, h, q, key]
    keep = mask.mean().item()
    assert abs(keep - (1 - p)) < 0.03, keep
    v = torch.randn(b, s, e, device=dev).to(BF)
    do = torch.randn(b, s, e, device=dev).to(BF)
    N.attn_fwd(q, k, v, e, e, e, 0, 0, 0, out, e, lse, None, b, s, h, dh, p, seed)
    dq, dk, dv = (torch.empty_like(q) for _ in range(3))
    N.attn_bwd(q, k, v, do, e, e, e, e, 0, 0, 0, 0, dq, dk, dv, e, e, e, 0, 0, 0, lse, None, b, s, h, dh, p, seed)
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    ref = _attn_ref(qr, kr, vr, h, None, mask, p)
    ref.backward(do.float())
    _close(out, ref, 2e-2, "out")
    for name, got, want in (("dq", dq, qr.grad), ("dk", dk, kr.grad), ("dv", dv, vr.grad)):
        _close(got, want, 4e-2, name)


def test_dropout_and_embeddings():
    _need()
    from split_learning_b200.ops import nn as F
    torch.manual_seed(4)
    x = torch.randn(64, 1024, device="cuda").to(BF).requires_grad_(True)
    y = F.dropout(x, 0.3, True)
    kept = (y != 0).float().mean().item()
    assert abs(kept - 0.7) < 0.02
    sel = y != 0
    _close(y[sel], (x / 0.7)[sel], 1e-2)
    y.backward(torch.ones_like(y))
    assert torch.equal(x.grad != 0, sel)
    vocab, d, b, s = 1000, 768, 4, 128
    word = torch.nn.Parameter(torch.randn(vocab, d, device="cuda"))
    pos = torch.nn.Parameter(torch.randn(512, d, device="cuda"))
    typ = torch.nn.Parameter(torch.randn(2, d, device="cuda"))
    ids = torch.randint(0, vocab, (b, s), device="cuda")
    ids[0, :5] = 0
    out = F.embed3(ids, None, word, pos, typ, 0)
    ref = word[ids] + pos[:s][None] + typ[0]
    _close(out, ref, 1e-2)
    g = torch.randn(b, s, d, device="cuda").to(BF)
    out.backward(g)
    wr = torch.zeros_like(word)
    wr.index_add_(0, ids.flatten(), g.float().view(-1, d))
    wr[0] = 0                                                              # padding_idx receives no gradient
    _close(word.grad, wr, 1e-3, "dword")
    _close(pos.grad[:s], g.float().sum(0), 1e-3, "dpos")
    _close(typ.grad[0], g.float().sum((0, 1)), 1e-3, "dtype")


def _stage_pair(name, data, start, end, batch):
    import copy
    from split_learning_b200.models import get_model_class
    from split_learning_b200.train.token_native import nativize
    torch.manual_seed(5)
    cls = get_model_class(name, data)
    ref = cls(start, end).cuda().eval()                 # eval(): dropout off on both sides, LN has no mode
    nat = nativize(copy.deepcopy(ref))
    if start == 0:
        x = cls.example_input(batch, device="cuda")
    else:
        with torch.no_grad():
            x = cls(0, start).cuda().eval()(cls.example_input(batch, device="cuda")).float()
    return ref, nat, x


@pytest.mark.parametrize("name,data,start,end,batch", [("KWT", "SPEECHCOMMANDS", 0, 17, 8), ("KWT", "SPEECHCOMMANDS", 5, 17, 8),
                                                        ("ViT", "CIFAR10", 0, 12, 8), ("ViT", "MNIST", 0, 12, 4),
                                                        ("BERT", "AGNEWS", 0, 3, 2), ("BERT", "AGNEWS", 11, 15, 2),
                                                        ("BERT", "EMOTION", 2, 6, 2)])
def test_native_stage_matches_torch(name, data, start, end, batch):
    _need()
    ref, nat, x = _stage_pair(name, data, start, end, batch)
    xr = x.clone().requires_grad_(True) if x.is_floating_point() else x
    xn = x.clone().requires_grad_(True) if x.is_floating_point() else x
    yr = ref(xr)
    yn = nat(xn).float()
    assert yn.shape == yr.shape
    assert _cos(yn, yr) > 0.995, _cos(yn, yr)
    g = torch.randn_like(yr)
    yr.backward(g)
    yn.backward(g)
    if x.is_floating_point():
        assert _cos(xn.grad, xr.grad) > 0.98, ("dx", _cos(xn.grad, xr.grad))
    bad = []
    for (k, pr), (_, pn) in zip(ref.named_parameters(), nat.named_parameters()):
        if pr.grad is None or pr.grad.abs().max() == 0:
            continue
        if "in_proj_bias" in k or k.endswith("key.bias"):
            continue                                     # the key bias has an exactly-zero gradient (softmax shift)
        c = _cos(pn.grad, pr.grad)
        if c < 0.97:
            bad.append((k, round(c, 4)))
    assert not bad, bad


def test_native_executor_trains_kwt():
    """Two KWT stages through TorchExecutor(native=True): the loss falls like the stock-torch executor's."""
    _need()
    from split_learning_b200.models import get_model_class
    from split_learning_b200.train.executor import TorchExecutor, make_executor
    cls = get_model_class("KWT", "SPEECHCOMMANDS")
    learning = {"learning-rate": 2e-3, "weight-decay": 0.01, "momentum": 0.5}
    losses = {}
    for native in (False, True):
        torch.manual_seed(7)
        m1, m2 = cls(0, 8), cls(8, 17)
        if native:
            e1 = make_executor(m1, "KWT", learning, "cuda", True, False)
            e2 = make_executor(m2, "KWT", learning, "cuda", False, True)
            assert e1.native and e2.native
        else:
            e1 = TorchExecutor(m1, "KWT", learning, "cuda", True, False)
            e2 = TorchExecutor(m2, "KWT", learning, "cuda", False, True)
        g = torch.Generator().manual_seed(11)
        x = torch.randn(16, 40, 98, generator=g)
        y = torch.randint(0, 10, (16,), generator=g)
        out = []
        for it in range(30):
            a = e1.forward_only(it, x)
            assert a.dtype == torch.float32
            gx = e2.forward_backward_last(a, y)
            e1.backward(it, gx)
            out.append(e2.last_loss())
        losses[native] = out
    assert losses[True][-1] < 0.6 * losses[True][0], losses[True]
    assert abs(losses[True][-1] - losses[False][-1]) < 0.5 * losses[False][0], (losses[True][-1], losses[False][-1])


def test_native_bert_lora_stage():
    """LoRA-wrapped BERT stage: only LoRA factors (and the classifier) receive gradients; merge still works."""
    _need()
    from split_learning_b200.models import get_model_class
    from split_learning_b200.models.lora import LoraConfig, apply_lora, merge_lora
    from split_learning_b200.train.token_native import nativize
    torch.manual_seed(9)
    cls = get_model_class("BERT", "AGNEWS")
    m = cls(12, 15).cuda()
    apply_lora(m, LoraConfig(), keep_trainable=("layer15",))
    nativize(m)
    m.train()
    x = torch.randn(2, 128, 768, device="cuda", requires_grad=True)
    out = m(x).float()
    assert out.shape == (2, 4)
    out.sum().backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()
    names = [k for k, p in m.named_parameters() if p.grad is not None and p.grad.abs().max() > 0]
    assert any("lora_B" in k or "lora_A" in k for k in names) and all(
        ("lora_" in k or "layer15" in k) for k in names), names
    merge_lora(m)
    assert all("lora" not in k for k in m.state_dict())


def test_graphed_steps_match_eager_and_redraw_dropout():
    """Whole-step CUDA graphs: same trajectory as the eager native path, fresh dropout masks on every replay, device-side
    AdamW step count."""
    _need()
    from split_learning_b200.models import get_model_class
    from split_learning_b200.train.executor import TorchExecutor
    cls = get_model_class("KWT", "SPEECHCOMMANDS")
    learning = {"learning-rate": 2e-3, "weight-decay": 0.01}
    g = torch.Generator().manual_seed(11)
    x = torch.randn(16, 40, 98, generator=g)
    y = torch.randint(0, 10, (16,), generator=g)
    finals = {}
    for graphs in (False, True):
        torch.manual_seed(7)
        e1 = TorchExecutor(cls(0, 8), "KWT", learning, "cuda", True, False, native=True, graphs=graphs)
        e2 = TorchExecutor(cls(8, 17), "KWT", learning, "cuda", False, True, native=True, graphs=graphs)
        for it in range(25):
            a = e1.forward_only(it, x)
            gx = e2.forward_backward_last(a, y)
            e1.backward(it, gx)
        finals[graphs] = e2.last_loss()
        if graphs:
            assert len(e1._graphs) == 2 and len(e2._graphs) == 1          # fwd + bwd, last
            assert int(e2.opt.dev_step.item()) == 25
            a1 = e1.forward_only("a", x)
            a2 = e1.forward_only("b", x)
            assert not torch.equal(a1, a2)                                # position dropout re-drawn per replay
            e1._store.clear()
    assert finals[True] < 1.2 and abs(finals[True] - finals[False]) < 0.6, finals
