"""Native eval-mode forward and server-side validation on it: the BatchNorm inference kernel, the loss / accuracy kernel,
the full-model evaluator against an fp64 torch oracle, determinism, stage composition, the resident test split and the
``b200.native-validation`` knob through ``run_inproc``."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LEARNING = {"learning-rate": 0.01, "momentum": 0.5, "batch-size": 32, "control-count": 3}


def _nrel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _row_cos(a, b):
    return F.cosine_similarity(a.double(), b.double(), dim=1)


# ----------------------------------------------------------------------------- shared model / data
@pytest.fixture(scope="module")
def trained():
    """VGG16_CIFAR10 whose BatchNorms hold real running statistics: a few seeded torch train-mode SGD steps."""
    from split_learning_b200.data import SyntheticDataset
    from split_learning_b200.models import VGG16_CIFAR10
    torch.manual_seed(0)
    model = VGG16_CIFAR10().to(DEV).train()
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.5)
    g = torch.Generator().manual_seed(1)
    ds = SyntheticDataset("CIFAR10", [32] * 10, seed=2)
    for _ in range(6):
        idx = torch.randint(0, len(ds), (32,), generator=g)
        x, y = ds.data[idx].to(DEV), ds.labels[idx].to(DEV)
        opt.zero_grad()
        F.cross_entropy(model(x), y).backward()
        opt.step()
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    ev = SyntheticDataset("CIFAR10", [105] * 10, seed=5)                 # 1,050 samples: 10 batches of 100 + one of 50
    perm = torch.randperm(1050, generator=torch.Generator().manual_seed(6))
    x, y = ev.data[perm], ev.labels[perm]
    batches = [(x[i:i + 100], y[i:i + 100]) for i in range(0, 1050, 100)]
    assert [b[0].shape[0] for b in batches] == [100] * 10 + [50]
    return sd, batches


def _torch_logits(sd, batches, dtype):
    from split_learning_b200.models import VGG16_CIFAR10
    m = VGG16_CIFAR10()
    m.load_state_dict(sd)
    m = m.to(DEV, dtype).eval()
    with torch.no_grad():
        return [m(x.to(DEV, dtype)).double() for x, _ in batches]


def _metrics(logits, batches):
    loss = sum(float(F.cross_entropy(lg, y.to(DEV))) for lg, (_, y) in zip(logits, batches)) / len(batches)
    correct = sum(int((lg.argmax(1) == y.to(DEV)).sum()) for lg, (_, y) in zip(logits, batches))
    return loss, correct


@pytest.fixture(scope="module")
def oracle(trained):
    sd, batches = trained
    return _torch_logits(sd, batches, torch.float64)


@pytest.fixture(scope="module")
def evaluator(trained):
    from split_learning_b200.models import VGG16_CIFAR10
    from split_learning_b200.train.b200_eval import NativeEvaluator
    sd, _ = trained
    return NativeEvaluator(VGG16_CIFAR10, sd, DEV)


def _check_against_oracle(m_native, logits_native, batches, oracle, yard):
    """Loss error <= 2 x the TF32 yardstick's + 1e-4; per-sample cosine no worse than the yardstick's - 1e-3; correct
    counts differ only on samples whose oracle top-2 margin is < 1e-3."""
    lo, co = _metrics(oracle, batches)
    ly, _ = _metrics(yard, batches)
    assert abs(m_native["val_loss"] - lo) <= 2 * abs(ly - lo) + 1e-4, (m_native["val_loss"], lo, ly)
    ref, nat, yd = torch.cat(oracle), torch.cat(logits_native), torch.cat(yard)
    assert float(_row_cos(nat, ref).min()) >= float(_row_cos(yd, ref).min()) - 1e-3
    labels = torch.cat([y for _, y in batches]).to(DEV)
    top2 = ref.topk(2, dim=1).values
    ambiguous = (top2[:, 0] - top2[:, 1]) < 1e-3
    differ = (nat.argmax(1) == labels) != (ref.argmax(1) == labels)
    assert not bool((differ & ~ambiguous).any())
    assert abs(m_native["val_correct"] - co) <= int(ambiguous.sum())
    assert m_native["val_total"] == labels.numel()


# ----------------------------------------------------------------------------- 1. BatchNorm inference kernel
@pytest.mark.parametrize("B,C,H,W", [(4, 64, 32, 32), (8, 128, 16, 16), (4, 512, 4, 4), (8, 512, 2, 2)])
@pytest.mark.parametrize("pool", [False, True])
@pytest.mark.parametrize("relu", [False, True])
def test_bn_infer_kernel(B, C, H, W, pool, relu):
    from split_learning_b200.ops import native as N
    N.preload(DEV)
    g = torch.Generator(device=DEV).manual_seed(B * C + H)
    y = torch.randn(B, H, W, C, device=DEV, generator=g) * 3.0 + 0.5
    gamma = torch.rand(C, device=DEV, generator=g) + 0.5
    beta = torch.randn(C, device=DEV, generator=g)
    rm = torch.randn(C, device=DEV, generator=g)
    rv = torch.rand(C, device=DEV, generator=g) * 4.0 + 0.25
    nbt = torch.tensor(17, device=DEV, dtype=torch.int64)
    before = [t.clone() for t in (rm, rv, nbt)]
    out = torch.empty(B, H // 2 if pool else H, W // 2 if pool else W, C, device=DEV)
    N.bn_relu_pool_infer(y, gamma, beta, rm, rv, out, H, W, relu, pool)
    torch.cuda.synchronize()
    ref = F.batch_norm(y.permute(0, 3, 1, 2), rm.clone(), rv.clone(), gamma, beta, training=False, eps=1e-5)
    if relu:
        ref = F.relu(ref)
    if pool:
        ref = F.max_pool2d(ref, 2)
    assert _nrel(out.permute(0, 3, 1, 2), ref) <= 1e-5
    assert all(torch.equal(a, b) for a, b in zip((rm, rv, nbt), before))


# ----------------------------------------------------------------------------- 2. loss / accuracy kernel
def _metric_case(B, seed, nan_row=False):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, 10, generator=g) * 3.0
    labels = torch.randint(0, 10, (B,), generator=g)
    logits[0, 3] = logits[0, 7] = 50.0          # tie: the first index wins
    labels[0] = 3
    logits[1, 2] = 60.0                         # tie with a different label: not correct
    logits[1, 6] = 60.0
    labels[1] = 6
    if nan_row:
        logits[2, 5] = float("nan")             # NaN counts as the maximum
        labels[2] = 5
    return logits, labels


@pytest.mark.parametrize("nan_row", [False, True])
def test_eval_metrics_kernel(nan_row):
    from split_learning_b200.ops import native as N
    N.preload(DEV)
    acc = torch.zeros(4, dtype=torch.float64, device=DEV)
    ints = acc.view(torch.int64)
    cases = [_metric_case(100, 1, nan_row), _metric_case(50, 2, nan_row)]
    for lg, lb in cases:
        N.eval_metrics(lg.to(DEV), lb.to(DEV), acc[0:1], ints[1:2], ints[2:3])
    torch.cuda.synchronize()
    want_loss = sum(float(F.cross_entropy(lg.double(), lb)) for lg, lb in cases)
    want_correct = sum(int((lg.argmax(1) == lb).sum()) for lg, lb in cases)
    assert int(ints[1]) == want_correct and int(ints[2]) == 150
    if nan_row:
        assert float(acc[0]) != float(acc[0])
    else:
        assert abs(float(acc[0]) - want_loss) <= 1e-6 * abs(want_loss)
    assert all(bool(lg[0].argmax() == 3) and bool(lg[1].argmax() == 2) for lg, _ in cases)


# ----------------------------------------------------------------------------- 3. whole model
def test_whole_model_against_fp64_oracle(trained, oracle, evaluator):
    sd, batches = trained
    yard = _torch_logits(sd, batches, torch.float32)                  # cuDNN TF32 convolutions: the reference's default
    m = evaluator.evaluate(batches)
    logits = [evaluator.logits(x).double() for x, _ in batches]
    _check_against_oracle(m, logits, batches, oracle, yard)


# ----------------------------------------------------------------------------- 4. determinism, no side effects
def test_deterministic_and_side_effect_free(trained, evaluator):
    sd, batches = trained
    before = {k: v.clone() for k, v in sd.items()}
    stats0 = evaluator.ex.S.clone(), evaluator.ex.P.clone()
    m1 = evaluator.evaluate(batches)
    l1 = [evaluator.logits(x) for x, _ in batches]
    m2 = evaluator.evaluate(batches)
    l2 = [evaluator.logits(x) for x, _ in batches]
    assert m1 == m2
    assert all(torch.equal(a, b) for a, b in zip(l1, l2))
    assert all(torch.equal(sd[k], before[k]) for k in sd)
    assert torch.equal(evaluator.ex.S, stats0[0]) and torch.equal(evaluator.ex.P, stats0[1])
    out = evaluator.ex.state_dict()
    assert all(torch.equal(out[k].cpu(), before[k]) for k in before)               # num_batches_tracked included
    assert evaluator.ex.G is None and evaluator.ex.M is None and evaluator.ex.PB is None and evaluator.ex.P_handle is None


# ----------------------------------------------------------------------------- 5. stage composition
def _stage(cls, a, b, sd, **kw):
    from split_learning_b200.train.b200_executor import B200Executor
    with torch.device("meta"):
        m = cls(a, b)
    keys = m.state_dict().keys()
    return B200Executor(cls(a, b), "VGG16", LEARNING, DEV, state_dict={k: sd[k] for k in keys}, **kw)


def test_stage_composition_and_training_untouched(trained, evaluator):
    from split_learning_b200.models import VGG16_CIFAR10
    from split_learning_b200.parallel.pipeline import LocalPipeline
    sd, batches = trained
    s1 = _stage(VGG16_CIFAR10, 0, 7, sd, is_first=True)
    s2 = _stage(VGG16_CIFAR10, 7, 52, sd, is_last=True)
    whole_bf16 = _stage(VGG16_CIFAR10, 0, 52, sd, is_first=True, is_last=True, precision="bf16")
    for x, _ in batches[-2:]:                                                    # a full and the short batch
        want = evaluator.logits(x)
        assert torch.equal(s2.eval_forward(s1.eval_forward(x)), want)
        assert torch.equal(whole_bf16.eval_forward(x), want)                    # eval is tf32 whatever the precision
    # training after eval_forward == training without it
    g = torch.Generator().manual_seed(9)
    data = [(torch.randn(32, 3, 32, 32, generator=g), torch.randint(0, 10, (32,), generator=g)) for _ in range(3)]
    runs = []
    for with_eval in (True, False):
        a = _stage(VGG16_CIFAR10, 0, 7, sd, is_first=True)
        b = _stage(VGG16_CIFAR10, 7, 52, sd, is_last=True)
        if with_eval:
            snap = [a.S.clone(), b.S.clone(), a.step_ctr.clone(), b.nan_flag.clone(),
                    [st["num_batches_tracked"].clone() for st in a.bn_state.values()]]
            b.eval_forward(a.eval_forward(data[0][0]))
            assert torch.equal(a.S, snap[0]) and torch.equal(b.S, snap[1])
            assert torch.equal(a.step_ctr, snap[2]) and torch.equal(b.nan_flag, snap[3])
            assert all(torch.equal(st["num_batches_tracked"], n) for st, n in zip(a.bn_state.values(), snap[4]))
            assert not a._store and not a.plans
        pipe = LocalPipeline([a, b], 32, 3)
        for x, y in data:
            pipe.run([(x, y)])
            pipe.synchronize()
        runs.append((float(pipe.loss()[0]), a.state_dict(), b.state_dict()))
    (la, a1, b1), (lb, a2, b2) = runs
    assert la == lb
    assert all(torch.equal(a1[k], a2[k]) for k in a1) and all(torch.equal(b1[k], b2[k]) for k in b1)


# ----------------------------------------------------------------------------- 6. resident uint8 path
def test_resident_uint8_matches_reference_normalisation(evaluator):
    from split_learning_b200.data.gpu_loader import CIFAR_MEAN, CIFAR_STD, GpuImageLoader, reference_batch
    g = torch.Generator().manual_seed(11)
    imgs = torch.randint(0, 256, (250, 32, 32, 3), generator=g, dtype=torch.uint8)
    labels = torch.randint(0, 10, (250,), generator=g)
    src = GpuImageLoader(imgs, labels, 100, DEV, CIFAR_MEAN, CIFAR_STD, augment=False, shuffle=False)
    m_res = evaluator.evaluate(src)
    z = torch.zeros(250, dtype=torch.int32)
    ref = reference_batch(imgs.to(DEV), torch.arange(250, device=DEV), z, z, z, CIFAR_MEAN, CIFAR_STD)
    m_ref = evaluator.evaluate([(ref[i:i + 100], labels[i:i + 100]) for i in range(0, 250, 100)])
    assert m_res["val_total"] == m_ref["val_total"] == 250
    assert m_res["val_correct"] == m_ref["val_correct"]
    assert abs(m_res["val_loss"] - m_ref["val_loss"]) <= 1e-6 * max(1.0, abs(m_ref["val_loss"]))


def test_resident_synthetic_split_matches_data_loader():
    from split_learning_b200.data import data_loader, resident_test_loader
    res = list(resident_test_loader("CIFAR10", DEV, synthetic=True))
    ref = list(data_loader("CIFAR10", train=False, synthetic=True))
    assert len(res) == len(ref)
    for (xr, yr), (xt, yt) in zip(res, ref):
        assert xr.is_cuda and torch.equal(xr.cpu(), xt) and torch.equal(yr.cpu(), yt)


# ----------------------------------------------------------------------------- 7. public API
def test_run_inproc_native_validation(tmp_path, monkeypatch):
    import yaml
    monkeypatch.setenv("SLB200_WAIT_SPINS", str(1 << 23))
    from split_learning_b200.checkpoint import load_checkpoint
    from split_learning_b200.config import normalize
    from split_learning_b200.data import data_loader
    from split_learning_b200.runner import run_inproc
    from split_learning_b200.validation import get_val
    raw = yaml.safe_load(open("config.yaml"))
    raw["server"].update({"clients": [1, 1], "global-round": 2, "validation": True})
    raw["server"]["data-distribution"]["num-sample"] = 320
    raw["log_path"] = str(tmp_path)
    raw["learning"].update({"batch-size": 32, "control-count": 3, "learning-rate": 0.01})
    raw["b200"] = {"synthetic-data": True, "watchdog-seconds": 120, "native-validation": True}
    monkeypatch.setenv("SLB200_SYNTHETIC", "1")
    srv = run_inproc(normalize(raw), devices=["cuda:0"], workdir=str(tmp_path), timeout=600)
    assert [h["ok"] for h in srv.history] == [True, True]
    assert all(h["val_backend"] == "native" for h in srv.history)
    sd = load_checkpoint(str(tmp_path / "VGG16_CIFAR10.pth"))                 # the last round's merged model
    ok, m_torch = get_val("VGG16", "CIFAR10", sd, device="cuda:0", synthetic=True)
    assert ok and m_torch["val_backend"] == "torch"
    batches = list(data_loader("CIFAR10", train=False, synthetic=True))
    oracle = _torch_logits(sd, batches, torch.float64)
    lo, co = _metrics(oracle, batches)
    top2 = torch.cat(oracle).topk(2, dim=1).values
    ambiguous = int(((top2[:, 0] - top2[:, 1]) < 1e-3).sum())
    last = srv.history[-1]
    assert last["val_total"] == m_torch["val_total"]
    assert abs(last["val_loss"] - lo) <= 2 * abs(m_torch["val_loss"] - lo) + 1e-4
    assert abs(last["val_correct"] - co) <= ambiguous
