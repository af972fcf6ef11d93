"""Native token-model validation on the GPU: the eval-only kernels against plain torch (and their host-side refusals), the
ViT / BERT eval programs graph-captured against the same program run eagerly, against an fp64 torch oracle of the same
state-dict, and ``b200.native-validation`` through ``get_val`` and ``run_inproc``.

Error bounds of the whole programs.  Every activation between kernels is bf16 (unit roundoff u = 2^-8) and the GEMM weights
are bf16 copies; a block of the programs rounds ~6 times (LayerNorm, QKV, attention, projection + residual, MLP), each a
relative error <= u that adds in quadrature over the blocks: sqrt(6 * 12) * u ~= 0.033 for BERT's 12 layers, 0.019 for
ViT's 6.  The per-batch norm-relative logit error is therefore held to 2^-4 (~2x the BERT estimate).  A prediction may
only flip where that error can swap the top two logits: the fp64 top-2 margin is below delta = 2 * 2^-4 * max|logit| of
the row.  The mean loss moves by at most max|d logit| per sample (cross-entropy is 1-Lipschitz in each logit's
difference to the log-sum-exp, up to 2x), so it is held to 2^-4 relative as well."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
BOUND = 2.0 ** -4


def _N():
    from split_learning_b200.ops import native as N
    N.preload(DEV)
    return N


# ----------------------------------------------------------------------------- 1. eval-only kernels
@pytest.mark.parametrize("B", [100, 7, 1])
def test_patch_rows_and_tokens(B):
    N = _N()
    g = torch.Generator(device=DEV).manual_seed(B)
    x = torch.randn(B, 3, 32, 32, device=DEV, generator=g)
    pt = torch.full((B * 64, 48), 7.0, dtype=torch.bfloat16, device=DEV)
    N.patch_rows(x, pt, 4)
    ref = x.reshape(B, 3, 8, 4, 8, 4).permute(0, 2, 4, 1, 3, 5).reshape(B * 64, 48).to(torch.bfloat16)
    assert torch.equal(pt, ref)
    pe = torch.randn(B * 64, 128, device=DEV, generator=g).to(torch.bfloat16)
    cls = torch.randn(128, device=DEV, generator=g)
    pos = torch.randn(65, 128, device=DEV, generator=g)
    out = torch.empty(B * 65, 128, dtype=torch.bfloat16, device=DEV)
    N.vit_tokens(pe, cls, pos, out, B, 64, 128)
    want = (torch.cat([cls.expand(B, 1, 128), pe.view(B, 64, 128)], dim=1) + pos).to(torch.bfloat16)
    assert torch.equal(out.view(B, 65, 128), want)


@pytest.mark.parametrize("B,S,D", [(100, 65, 128), (7, 65, 128), (1, 128, 768), (33, 3, 2)])
def test_ln_rows_matches_ln_fwd_and_torch(B, S, D):
    N = _N()
    g = torch.Generator(device=DEV).manual_seed(B * S + D)
    x = (torch.randn(B * S, D, device=DEV, generator=g) * 3.0 + 1.0).to(torch.bfloat16)
    gamma = torch.rand(D, device=DEV, generator=g) + 0.5
    beta = torch.randn(D, device=DEV, generator=g)
    y = torch.empty(B, D, dtype=torch.bfloat16, device=DEV)
    N.ln_rows_fwd(x, S * D, gamma, beta, y, B, D, 1e-5)
    rows = x.view(B, S, D)[:, 0].contiguous()
    y2 = torch.empty_like(y)
    mean, rstd = torch.empty(B, device=DEV), torch.empty(B, device=DEV)
    N.ln_fwd(rows, None, gamma, beta, y2, None, mean, rstd, B, D, 1e-5)
    assert torch.equal(y, y2)                                                 # the same bits as the training LayerNorm
    ref = F.layer_norm(rows.double(), (D,), gamma.double(), beta.double(), 1e-5)
    assert float((y.double() - ref).abs().max()) <= 2.0 ** -7 * float(ref.abs().max()) + 1e-6


@pytest.mark.parametrize("M,N_,K,lda", [(100, 10, 128, 128), (7, 4, 768, 768), (1, 4, 768, 128 * 768), (20, 4, 768, 128 * 768),
                                        (50, 100, 64, 72)])
def test_gemm_bias_f32(M, N_, K, lda):
    N = _N()
    g = torch.Generator(device=DEV).manual_seed(M * N_ + K)
    a_store = torch.randn(M, lda, device=DEV, generator=g).to(torch.bfloat16)
    a = a_store[:, :K]
    w = torch.randn(N_, K, device=DEV, generator=g).to(torch.bfloat16)
    bias = torch.randn(N_, device=DEV, generator=g)
    out = torch.full((M + 1, N_), 5.0, device=DEV)                             # one guard row after the output
    N.gemm_bias_f32(a_store, w, out, bias, M, N_, K, lda=lda)
    ref = a.double() @ w.double().T + bias.double()
    scale = a.double().abs() @ w.double().abs().T + bias.double().abs()
    assert bool(((out[:M].double() - ref).abs() <= 2.0 ** -20 * K * scale).all())
    assert bool((out[M] == 5.0).all())
    again = torch.empty(M, N_, device=DEV)
    N.gemm_bias_f32(a_store, w, again, bias, M, N_, K, lda=lda)
    assert torch.equal(again, out[:M])


def test_host_checks_refuse_before_launch():
    N = _N()
    x = torch.randn(2, 3, 30, 32, device=DEV)
    pt = torch.full((2 * 56, 48), 3.0, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(N.NativeError):
        N.patch_rows(x, pt, 4)                                                # 30 % 4 != 0
    with pytest.raises(N.NativeError):
        N.patch_rows(torch.randn(2, 1, 8, 8, device=DEV), pt, 2)              # K = 4 is not a multiple of 8
    pe = torch.zeros(2 * 4, 6, dtype=torch.bfloat16, device=DEV)
    out = torch.full((2 * 5, 7), 3.0, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(N.NativeError):
        N.vit_tokens(pe, torch.zeros(7, device=DEV), torch.zeros(5, 7, device=DEV), out, 2, 4, 7)   # odd E
    xs = torch.zeros(4, 64, dtype=torch.bfloat16, device=DEV)
    y = torch.full((4, 64), 3.0, dtype=torch.bfloat16, device=DEV)
    ones = torch.ones(64, device=DEV)
    with pytest.raises(N.NativeError):
        N.ln_rows_fwd(xs, 32, ones, ones, y, 4, 64, 1e-5)                     # pitch < D
    with pytest.raises(N.NativeError):
        N.ln_rows_fwd(xs, 65, ones, ones, y, 4, 64, 1e-5)                     # odd pitch
    a = torch.zeros(4, 60, dtype=torch.bfloat16, device=DEV)
    w = torch.zeros(4, 60, dtype=torch.bfloat16, device=DEV)
    o = torch.full((4, 4), 3.0, device=DEV)
    with pytest.raises(N.NativeError):
        N.gemm_bias_f32(a, w, o, torch.zeros(4, device=DEV), 4, 4, 60)        # K % 8 != 0
    with pytest.raises(N.NativeError):
        N.gemm_bias_f32(a[:, :56], w[:, :56], o, None, 4, 4, 56, lda=60, ldb=60)   # no bias
    torch.cuda.synchronize()
    assert bool((pt == 3.0).all()) and bool((out == 3.0).all()) and bool((y == 3.0).all()) and bool((o == 3.0).all())


# ----------------------------------------------------------------------------- 2. whole programs
def _train(model, batches, lr):
    opt = torch.optim.AdamW(model.parameters(), lr=lr)
    for x, y, kw in batches:
        opt.zero_grad()
        F.cross_entropy(model(**kw) if kw else model(x), y).backward()
        opt.step()


@pytest.fixture(scope="module")
def vit():
    from split_learning_b200.data import SyntheticDataset
    from split_learning_b200.models import ViT_CIFAR10
    torch.manual_seed(0)
    m = ViT_CIFAR10().to(DEV).train()
    ds = SyntheticDataset("CIFAR10", [16] * 10, seed=3)
    g = torch.Generator().manual_seed(4)
    steps = []
    for _ in range(4):
        idx = torch.randint(0, len(ds), (32,), generator=g)
        steps.append((ds.data[idx].to(DEV), ds.labels[idx].to(DEV), None))
    _train(m, steps, 1e-3)
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    ev = SyntheticDataset("CIFAR10", [25] * 10, seed=5)                       # 250 samples: 100, 100, 50
    batches = [(ev.data[i:i + 100], ev.labels[i:i + 100]) for i in range(0, 250, 100)]
    return ViT_CIFAR10, sd, batches, [100, 50, 1]


@pytest.fixture(scope="module")
def bert():
    from split_learning_b200.data import SyntheticDataset
    from split_learning_b200.models import BERT_AGNEWS
    torch.manual_seed(1)
    m = BERT_AGNEWS().to(DEV).train()
    ds = SyntheticDataset("AGNEWS", [8] * 4, seed=3)
    steps = [(None, ds.labels[i:i + 4].to(DEV), {"input_ids": ds.data[i:i + 4].to(DEV)}) for i in (0, 8, 16)]
    _train(m, steps, 1e-4)
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    ev = SyntheticDataset("AGNEWS", [12] * 4, seed=5)                         # 48 samples: 20, 20, 8
    batches = [(ev.data[i:i + 20], ev.labels[i:i + 20]) for i in range(0, 48, 20)]
    return BERT_AGNEWS, sd, batches, [20, 7, 1]


@pytest.fixture(params=["vit", "bert"])
def case(request):
    return request.getfixturevalue(request.param)


def _oracle(cls, sd, x):
    m = cls()
    m.load_state_dict(sd)
    m = m.to(DEV, torch.float64).eval()
    with torch.no_grad():
        if x.dtype == torch.long:
            return m(input_ids=x.to(DEV))
        return m(x.to(DEV, torch.float64))


def test_graph_equals_eager_program(case):
    from split_learning_b200.train.token_eval import NativeTokenEvaluator
    cls, sd, batches, sizes = case
    graphed = NativeTokenEvaluator(cls, sd, DEV)
    eager = NativeTokenEvaluator(cls, sd, DEV, use_graphs=False)
    x_all = torch.cat([x for x, _ in batches])
    for b in sizes:
        x = x_all[:b]
        want = eager.logits(x)
        runs = [graphed.logits(x) for _ in range(4)]                          # eager warm-up, capture, two replays
        assert len(graphed.plans[tuple(x.shape)].graphs) == 1
        assert all(torch.equal(r, want) for r in runs), b
        assert want.dtype == torch.float32 and want.shape == (b, cls.num_classes())
    assert graphed.evaluate(batches) == eager.evaluate(batches) == graphed.evaluate(batches)


def test_program_against_fp64_oracle(case):
    from split_learning_b200.train.token_eval import NativeTokenEvaluator
    cls, sd, batches, _ = case
    ev = NativeTokenEvaluator(cls, sd, DEV)
    m = ev.evaluate(batches)
    nat, ref = [], []
    for x, _ in batches:
        lg, rf = ev.logits(x).double(), _oracle(cls, sd, x)
        rel = float((lg - rf).norm() / rf.norm())
        assert rel <= BOUND, rel
        nat.append(lg)
        ref.append(rf)
    nat, ref = torch.cat(nat), torch.cat(ref)
    labels = torch.cat([y for _, y in batches]).to(DEV)
    top2 = ref.topk(2, dim=1).values
    ambiguous = (top2[:, 0] - top2[:, 1]) < 2 * BOUND * ref.abs().max(dim=1).values
    differ = (nat.argmax(1) == labels) != (ref.argmax(1) == labels)
    assert not bool((differ & ~ambiguous).any())
    co = int((ref.argmax(1) == labels).sum())
    assert abs(m["val_correct"] - co) <= int(ambiguous.sum()) and m["val_total"] == labels.numel()
    lo = sum(float(F.cross_entropy(r, y.to(DEV))) for r, (_, y) in zip(ref.split([x.shape[0] for x, _ in batches]), batches))
    lo /= len(batches)
    assert abs(m["val_loss"] - lo) <= BOUND * abs(lo), (m["val_loss"], lo)


def test_reload_keeps_graphs_valid(vit):
    from split_learning_b200.train.token_eval import NativeTokenEvaluator
    cls, sd, batches, _ = vit
    ev = NativeTokenEvaluator(cls, sd, DEV)
    m1 = ev.evaluate(batches)
    ev.evaluate(batches)                                                      # graphs captured
    sd2 = {k: v * 0.5 if v.is_floating_point() else v for k, v in sd.items()}
    ev.load_state_dict(sd2)
    fresh = NativeTokenEvaluator(cls, sd2, DEV, use_graphs=False)
    assert ev.evaluate(batches) == fresh.evaluate(batches) != m1


def test_bert_emotion_program():
    from split_learning_b200.models import BERT_EMOTION
    from split_learning_b200.train.token_eval import NativeTokenEvaluator
    torch.manual_seed(2)
    sd = BERT_EMOTION().state_dict()
    x = torch.randint(1, BERT_EMOTION.VOCAB, (7, 128))
    lg = NativeTokenEvaluator(BERT_EMOTION, sd, DEV).logits(x).double()
    rf = _oracle(BERT_EMOTION, sd, x)
    assert float((lg - rf).norm() / rf.norm()) <= BOUND


# ----------------------------------------------------------------------------- 3. public API
def test_get_val_native_and_cache(bert):
    from split_learning_b200 import validation as V
    from split_learning_b200.train.token_eval import NativeTokenEvaluator
    _, sd, _, _ = bert
    V._NATIVE.clear()
    ok, m1 = V.get_val("BERT", "AGNEWS", sd, device="cuda:0", synthetic=True, native=True)
    assert ok and m1["val_backend"] == "native" and m1["val_total"] == 100
    (ev, src), = V._NATIVE.values()
    assert isinstance(ev, NativeTokenEvaluator)
    ok, m2 = V.get_val("BERT", "AGNEWS", sd, device="cuda:0", synthetic=True, native=True)
    assert m2 == m1 and list(V._NATIVE.values())[0][0] is ev
    ok, mt = V.get_val("BERT", "AGNEWS", sd, device="cuda:0", synthetic=True, native=False)
    assert mt["val_backend"] == "torch" and mt["val_total"] == m1["val_total"]
    V._NATIVE.clear()


@pytest.mark.parametrize("cfg,labels", [("configs/vit_cifar10.yaml", 10), ("configs/bert_agnews.yaml", 4)])
def test_run_inproc_native_validation_auto(tmp_path, monkeypatch, cfg, labels):
    import yaml
    from split_learning_b200 import validation as V
    from split_learning_b200.config import normalize
    from split_learning_b200.runner import run_inproc
    from split_learning_b200.train.token_eval import NativeTokenEvaluator
    monkeypatch.setenv("SLB200_SYNTHETIC", "1")
    V._NATIVE.clear()
    made = []
    real = NativeTokenEvaluator.__init__

    def spy(self, *a, **k):
        real(self, *a, **k)
        made.append(self)
    monkeypatch.setattr(NativeTokenEvaluator, "__init__", spy)
    raw = yaml.safe_load(open(cfg))
    bs = raw["learning"]["batch-size"]
    raw["server"].update({"global-round": 2, "validation": True})
    raw["server"]["data-distribution"]["num-sample"] = 2 * bs * labels
    raw["log_path"] = str(tmp_path)
    raw["b200"].update({"native-validation": "auto", "watchdog-seconds": 120})
    srv = run_inproc(normalize(raw), devices=["cuda:0"], workdir=str(tmp_path), timeout=600)
    assert [h["ok"] for h in srv.history] == [True, True]
    assert all(h["val_backend"] == "native" for h in srv.history)
    assert len(made) == 1                                                     # the second round reused the evaluator
    V._NATIVE.clear()
