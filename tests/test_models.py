import pytest
import torch

from oracle_cases import layout_digest, load_json, model_cases

from split_learning_b200.models import (BERT_AGNEWS, BERT_EMOTION, KWT_SPEECHCOMMANDS, MobileNetv1_CIFAR10,
                                        VGG16_CIFAR10, VGG16_MNIST, ViT_CIFAR10, ViT_MNIST, build_stage,
                                        get_model_class)
from split_learning_b200.models.lora import apply_lora, merge_lora

# state-dict layouts and forward outputs of the reference model classes (src/model/*.py, other/Vanilla_SL/src/model/*.py),
# recorded by tools/make_golden.py
ORACLE = load_json("models.json")
CASES = [(c[0], c[2]) for c in model_cases()]


@pytest.mark.parametrize("mine,cls", CASES, ids=[c[1] for c in CASES])
def test_state_dict_keys_match_reference(mine, cls):
    n = mine.num_layers()
    for a, b in [(0, n), (0, 3), (3, n), (2, 5)]:
        # same keys in the same order, same shapes and dtypes (stored as a digest of the reference's list)
        assert layout_digest(mine(a, b).state_dict()) == ORACLE["layouts"][cls][f"{a},{b}"], (cls, a, b)


@pytest.mark.parametrize("mine,cls", [CASES[0], CASES[1], CASES[5]], ids=["VGG16", "KWT", "ViT"])
def test_forward_matches_reference(mine, cls):
    # the recorded outputs are the reference model's, run with the weights our class draws under seed 0
    torch.manual_seed(0)
    m = mine().eval()
    torch.manual_seed(1)
    x = mine.example_input(2)
    with torch.no_grad():
        assert torch.allclose(m(x), torch.tensor(ORACLE["forward"][cls]), atol=1e-5)


def test_vgg16_table_facts():
    m = VGG16_CIFAR10()
    sd = m.state_dict()
    assert len(sd) == 97
    assert sum(p.numel() for p in m.parameters()) == 33_646_666
    assert sum(1 for v in sd.values() if v.dtype == torch.int64) == 13
    s1, s2 = VGG16_CIFAR10(0, 7), VGG16_CIFAR10(7, 52)
    assert set(s1.state_dict()) | set(s2.state_dict()) == set(sd)
    assert not set(s1.state_dict()) & set(s2.state_dict())
    x = torch.randn(4, 3, 32, 32)
    assert s1(x).shape == (4, 64, 16, 16)
    assert s2(s1(x)).shape == (4, 10)


def test_stage_composition_equals_full():
    torch.manual_seed(0)
    full = VGG16_CIFAR10().eval()
    parts = [VGG16_CIFAR10(0, 5).eval(), VGG16_CIFAR10(5, 10).eval(), VGG16_CIFAR10(10, 52).eval()]
    for p in parts:
        p.load_state_dict({k: full.state_dict()[k] for k in p.state_dict()})
    x = torch.randn(2, 3, 32, 32)
    y = x
    for p in parts:
        y = p(y)
    assert torch.allclose(y, full(x), atol=1e-5)


def test_build_stage_conventions():
    assert build_stage("VGG16", "CIFAR10", [0, 7]).end_layer == 7
    assert build_stage("VGG16", "CIFAR10", [7, -1]).start_layer == 7
    whole = build_stage("VGG16", None, [0, 0])
    assert (whole.start_layer, whole.end_layer) == (0, 52)
    assert get_model_class("KWT").__name__ == "KWT_SPEECHCOMMANDS"
    with pytest.raises(ValueError):
        get_model_class("nope")


def test_lora_roundtrip():
    torch.manual_seed(0)
    m = BERT_AGNEWS(12, 15)
    keys = list(m.state_dict())
    x = torch.randn(2, 8, 768)
    apply_lora(m, keep_trainable=("layer15.classifier",))
    trainable = [n for n, p in m.named_parameters() if p.requires_grad]
    assert any("lora_A" in n for n in trainable) and any("layer15.classifier" in n for n in trainable)
    assert not any(n.endswith("base.weight") for n in trainable)
    for n, p in m.named_parameters():
        if "lora_B" in n:
            torch.nn.init.normal_(p, std=0.02)
    m.eval()
    y = m(x)
    merge_lora(m)
    assert list(m.state_dict()) == keys
    assert torch.allclose(m(x), y, atol=1e-5)


def test_native_rebinding_keeps_module_tree():
    """``nativize`` only re-binds ``forward`` attributes (state-dict keys, LoRA wrapping / merging unaffected);
    ``cnn_native._program`` groups conv / BN / ReLU / pool runs of any cut correctly."""
    from split_learning_b200.models.lora import LoraConfig, apply_lora, merge_lora
    from split_learning_b200.train import cnn_native, token_native
    m = BERT_AGNEWS(12, 15)
    keys = list(m.state_dict())
    apply_lora(m, LoraConfig(), keep_trainable=("layer15",))
    token_native.nativize(m)
    assert any("lora_A" in k for k in m.state_dict())
    merge_lora(m)
    assert list(m.state_dict()) == keys
    token_native.denativize(m)
    assert m(torch.randn(1, 128, 768)).shape == (1, 4)               # stock forward restored (CPU)
    k = KWT_SPEECHCOMMANDS(0, 17)
    token_native.nativize(k)
    assert "forward" in k.layer4.__dict__ and "forward" in k.layer16.__dict__ and list(k.state_dict()) == list(
        KWT_SPEECHCOMMANDS(0, 17).state_dict())
    assert cnn_native.supports(MobileNetv1_CIFAR10(0, 3)) and not cnn_native.supports(k)
    prog = cnn_native._program(MobileNetv1_CIFAR10(0, 84))
    assert prog[0] == ("stem", 1) and prog[1] == ("bn", 2, True, False) and prog[-3:] == [("bn", 80, True, True), ("flatten",),
                                                                                           ("linear", 84)]
    assert sum(1 for op in prog if op[0] == "conv3") == 13 and sum(1 for op in prog if op[0] == "conv1") == 13
    assert cnn_native._program(MobileNetv1_CIFAR10(2, 5)) == [("relu",), ("conv3", 4), ("bn", 5, False, False)]
