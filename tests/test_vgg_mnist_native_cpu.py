"""VGG16_MNIST routing: the cnn_native stage program takes it, the compiled VGG plan keeps refusing it."""
from split_learning_b200.models import VGG16_CIFAR10, VGG16_MNIST
from split_learning_b200.train import b200_executor, cnn_native


def test_cnn_native_supports_vgg16_mnist_only():
    assert cnn_native.supports(VGG16_MNIST())
    assert cnn_native.supports(VGG16_MNIST(0, 7)) and cnn_native.supports(VGG16_MNIST(7, 51))
    assert not cnn_native.supports(VGG16_CIFAR10())


def test_compiled_plan_still_rejects_vgg16_mnist():
    assert not b200_executor.supports(VGG16_MNIST())
    assert b200_executor.supports(VGG16_CIFAR10())


def test_vgg16_mnist_program():
    ops = cnn_native._program(VGG16_MNIST(0, 51))
    block = lambda i, pool: [("conv3", i), ("bn", i + 1, True, pool)]      # noqa: E731
    expect = [("stem", 1), ("bn", 2, True, False)] + block(4, True)         # 28x28, pool -> 14
    expect += block(8, False) + block(11, True)                             # 14x14, pool -> 7
    expect += block(15, False) + block(18, False) + block(21, True)         # 7x7, pool -> 3
    expect += block(25, False) + block(28, False) + block(31, True)         # 3x3, pool -> 1
    expect += block(35, False) + block(38, False) + block(41, False)        # 1x1
    expect += [("flatten",), ("dropout", 45), ("linear", 46, "relu"), ("dropout", 48), ("linear", 49, "relu"),
               ("linear", 51)]
    assert ops == expect


def test_vgg16_mnist_stage_programs_cover_every_layer():
    for s, e in ((0, 7), (7, 14), (14, 24), (24, 34), (34, 44), (44, 51), (7, 51)):
        ops = cnn_native._program(VGG16_MNIST(s, e))
        assert ops, (s, e)
    assert cnn_native._program(VGG16_MNIST(44, 51))[0] == ("dropout", 45)
