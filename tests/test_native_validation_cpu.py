"""``b200.native-validation`` routing without a GPU: the default keeps the torch path, ``auto`` falls back to torch with
one log line giving the reason, ``true`` raises where there is no native plan, and the supports check on the meta device."""
import pytest
import torch


class _Log:
    def __init__(self):
        self.lines = []

    def log_info(self, s):
        self.lines.append(s)


@pytest.fixture
def no_cuda(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)


def _kwt_state():
    from split_learning_b200.models import get_model_class
    torch.manual_seed(0)
    return get_model_class("KWT", "SPEECHCOMMANDS")().state_dict()


def test_default_takes_torch(no_cuda):
    from split_learning_b200.validation import get_val
    log = _Log()
    ok, m = get_val("KWT", "SPEECHCOMMANDS", _kwt_state(), logger=log, device="cpu", synthetic=True)
    assert ok and m["val_backend"] == "torch" and m["val_total"] > 0
    assert not any("native" in s for s in log.lines)


@pytest.mark.parametrize("model,data", [("VGG16", "CIFAR10"), ("KWT", "SPEECHCOMMANDS")])
def test_auto_without_cuda_takes_torch_and_logs(no_cuda, monkeypatch, model, data):
    from split_learning_b200 import validation as V
    calls = []
    monkeypatch.setattr(V, "evaluate", lambda m, loader, device, pump=None: calls.append(device) or
                        {"val_loss": 1.0, "val_acc": 10.0, "val_correct": 1, "val_total": 10})
    log = _Log()
    from split_learning_b200.models import get_model_class
    sd = get_model_class(model, data)().state_dict()
    ok, m = V.get_val(model, data, sd, logger=log, synthetic=True, native="auto")
    assert ok and m["val_backend"] == "torch" and calls == ["cpu"]
    reasons = [s for s in log.lines if "native validation unavailable" in s]
    assert len(reasons) == 1 and "no CUDA device" in reasons[0]


def test_auto_with_kwt_names_the_model(monkeypatch):
    from split_learning_b200 import validation as V
    from split_learning_b200.models import get_model_class
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    reason = V.native_unsupported_reason(get_model_class("KWT", "SPEECHCOMMANDS"), "SPEECHCOMMANDS", "cuda:0")
    assert reason is not None and "SPEECHCOMMANDS" in reason
    reason = V.native_unsupported_reason(get_model_class("VGG16", "MNIST"), "CIFAR10", "cuda:0")
    assert reason == "VGG16_MNIST has no native eval plan"
    assert V.native_unsupported_reason(get_model_class("VGG16", "CIFAR10"), "CIFAR10", "cuda:0") is None


def test_true_without_cuda_raises(no_cuda):
    from split_learning_b200.validation import get_val
    with pytest.raises(RuntimeError, match="no CUDA device"):
        get_val("KWT", "SPEECHCOMMANDS", _kwt_state(), device="cpu", synthetic=True, native=True)


def test_knob_values():
    from split_learning_b200.config import DEFAULT_B200
    from split_learning_b200.validation import native_mode
    assert DEFAULT_B200["native-validation"] is False
    assert [native_mode(v) for v in (False, None, "false", True, "true", "auto", "AUTO")] == \
        ["false", "false", "false", "true", "true", "auto", "auto"]
    with pytest.raises(ValueError):
        native_mode("sometimes")


def test_supports_from_layer_tables_on_meta():
    from split_learning_b200.models import get_model_class
    from split_learning_b200.train.b200_eval import native_eval_supported
    assert native_eval_supported(get_model_class("VGG16", "CIFAR10"))
    assert not native_eval_supported(get_model_class("VGG16", "MNIST"))          # width 28 does not divide 128
    for model, data in [("KWT", "SPEECHCOMMANDS"), ("MobileNetv1", "CIFAR10"), ("ViT", "CIFAR10"), ("BERT", "AGNEWS")]:
        assert not native_eval_supported(get_model_class(model, data))
