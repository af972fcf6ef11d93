"""Every sm_90a kernel against a plain PyTorch fp32 reference (needs an H100)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def selftest():
    from split_learning_b200.ops import native, selftest
    native.require()
    return selftest


@pytest.mark.parametrize("name", ["conv_fwd_tf32", "conv_dgrad_tf32", "conv_wgrad_tf32", "fused_cut_tail_tf32", "linear_f32", "bn_fwd_bwd_f32",
                                  "conv1_direct_f32", "conv_fwd", "conv_dgrad", "conv_dgrad_bn_stats", "conv_wgrad", "fused_cut_tail",
                                  "linear_all", "bn_fwd_bwd", "conv1_direct", "ce_and_linear_epilogues", "optimizers_and_fedavg",
                                  "flags_and_peer"])
def test_kernel(selftest, name):
    err, tol = selftest.CHECKS[name]()
    assert err <= tol, f"{name}: err {err} > tol {tol}"


@pytest.mark.gpu
def test_gpu_image_loader_matches_reference_recipe():
    """image_batch_kernel == RandomCrop(32, 4) + HFlip + ToTensor + Normalize done with torch ops, and the loader yields a
    full epoch of device-resident microbatches."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from split_learning_b200.data.gpu_loader import CIFAR_MEAN, CIFAR_STD, GpuImageLoader, reference_batch
    g = torch.Generator().manual_seed(0)
    images = torch.randint(0, 256, (500, 32, 32, 3), generator=g, dtype=torch.uint8)
    labels = torch.randint(0, 10, (500,), generator=g)
    ld = GpuImageLoader(images, labels, 32, "cuda", CIFAR_MEAN, CIFAR_STD, seed=3)
    idx = torch.randperm(500, device="cuda")[:32]
    dx, dy, flip = ld.draw(32)
    assert int(dx.min()) >= -4 and int(dx.max()) <= 4 and set(flip.tolist()) <= {0, 1}
    x, y = ld.batch(idx, dx, dy, flip)
    ref = reference_batch(ld.images, idx, dx.tolist(), dy.tolist(), flip.tolist(), CIFAR_MEAN, CIFAR_STD)
    assert x.shape == (32, 3, 32, 32) and torch.allclose(x, ref, atol=1e-5)
    assert torch.equal(y, ld.labels[idx])
    seen = torch.cat([yy for _, yy in ld])
    assert len(ld) == 16 and seen.numel() == 500 and torch.equal(seen.sort().values, ld.labels.sort().values)
    mono = GpuImageLoader(images[..., :1].contiguous(), labels, 50, "cuda", (0.1307,), (0.3081,), augment=False, shuffle=False)
    xm, _ = next(iter(mono))
    assert torch.allclose(xm, (images[:50, :, :, :1].permute(0, 3, 1, 2).float().cuda() / 255 - 0.1307) / 0.3081, atol=1e-5)
