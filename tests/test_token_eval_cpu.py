"""Native token-model validation without a GPU: ``b200.native-validation`` routing for ViT, BERT and KWT, the token eval
predicate on the meta device, and the resident AGNEWS / EMOTION test splits against the host test loader."""
import pytest
import torch


class _Log:
    def __init__(self):
        self.lines = []

    def log_info(self, s):
        self.lines.append(s)


_M = {"val_loss": 1.0, "val_acc": 10.0, "val_correct": 1, "val_total": 10}
CASES = [("ViT", "CIFAR10", True), ("BERT", "AGNEWS", True), ("BERT", "EMOTION", True), ("KWT", "SPEECHCOMMANDS", False)]


@pytest.fixture
def routed(monkeypatch):
    """CUDA reported present; both backends replaced by recorders."""
    from split_learning_b200 import validation as V
    calls = []
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(V, "_native_evaluate", lambda klass, *a, **k: calls.append(("native", klass.__name__)) or dict(_M))
    monkeypatch.setattr(V, "evaluate", lambda m, loader, device, pump=None: calls.append(("torch", type(m).__name__))
                        or dict(_M))
    monkeypatch.setattr(V, "data_loader", lambda **k: [])
    monkeypatch.setattr(torch.nn.Module, "to", lambda self, *a, **k: self)      # the torch path's model.to("cuda:0")
    return V, calls


def _sd(model, data):
    from split_learning_b200.models import get_model_class
    with torch.device("meta"):
        m = get_model_class(model, data)()
    return {k: torch.zeros(v.shape, dtype=v.dtype) for k, v in m.state_dict().items()}


@pytest.mark.parametrize("model,data,native", CASES)
@pytest.mark.parametrize("mode", ["auto", "true", "false"])
def test_routing(routed, model, data, native, mode):
    V, calls = routed
    log = _Log()
    if mode == "true" and not native:
        with pytest.raises(RuntimeError, match="SPEECHCOMMANDS"):
            V.get_val(model, data, _sd(model, data), logger=log, device="cuda:0", synthetic=True, native=mode)
        assert calls == []
        return
    ok, m = V.get_val(model, data, _sd(model, data), logger=log, device="cuda:0", synthetic=True, native=mode)
    want = "native" if native and mode != "false" else "torch"
    assert ok and m["val_backend"] == want and [c[0] for c in calls] == [want]
    fallback = [s for s in log.lines if "native validation unavailable" in s]
    assert len(fallback) == (1 if (mode == "auto" and not native) else 0)


def test_unsupported_reasons(monkeypatch):
    from split_learning_b200 import validation as V
    from split_learning_b200.models import get_model_class
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    for model, data in [("ViT", "CIFAR10"), ("BERT", "AGNEWS"), ("BERT", "EMOTION")]:
        assert V.native_unsupported_reason(get_model_class(model, data), data, "cuda:0") is None
        assert V.native_unsupported_reason(get_model_class(model, data), data, "cpu") == "no CUDA device"
    assert V.native_unsupported_reason(get_model_class("ViT", "CIFAR10"), "AGNEWS", "cuda:0") == \
        "no resident test split for AGNEWS"
    assert V.native_unsupported_reason(get_model_class("ViT", "MNIST"), "MNIST", "cuda:0") == "no resident test split for MNIST"


def test_token_eval_predicate_on_meta():
    from split_learning_b200.models import get_model_class
    from split_learning_b200.train.b200_eval import native_eval_supported
    from split_learning_b200.train.token_eval import token_eval_supported
    yes = [("ViT", "CIFAR10"), ("BERT", "AGNEWS"), ("BERT", "EMOTION")]
    no = [("KWT", "SPEECHCOMMANDS"), ("ViT", "MNIST"), ("VGG16", "CIFAR10"), ("VGG16", "MNIST"), ("MobileNetv1", "CIFAR10")]
    for model, data in yes:
        assert token_eval_supported(get_model_class(model, data))
        assert not native_eval_supported(get_model_class(model, data))          # the VGG-plan predicate is unchanged
    for model, data in no:
        assert not token_eval_supported(get_model_class(model, data))


@pytest.mark.parametrize("name", ["AGNEWS", "EMOTION"])
def test_resident_text_split_matches_host_loader(name):
    from split_learning_b200.data import data_loader, resident_test_loader
    res = list(resident_test_loader(name, "cpu", synthetic=True))
    ref = list(data_loader(name, train=False, synthetic=True))
    assert len(res) == len(ref) > 0
    for (xr, yr), b in zip(res, ref):
        assert xr.dtype == torch.int64 and torch.equal(xr, b["input_ids"]) and torch.equal(yr, b["labels"])
    sizes = [x.shape[0] for x, _ in res]
    assert all(s == 20 for s in sizes[:-1]) and 1 <= sizes[-1] <= 20
