"""tf32 conv input and weight gradients (MN-major operands, transposed in shared memory before the MMAs) at every conv
shape of the self-test, at forced BLOCK_N and forced split-K, and on M tails:

* the result bits match SHA-256 digests committed in ``tests/golden/tf32_conv_backward_sha256.json`` (recorded from the
  kernels as they were before the in-place pipelined transpose: any change of a result bit shows up here);
* every result is within the tf32 tolerance of an fp64 oracle;
* repeated launches give the same bits;
* the cut-head dgrad captured with its mailbox publish in a CUDA graph replays to the eager bits.

``python tests/test_tf32_conv_backward_gpu.py --write PATH`` records the digests of the current kernels."""
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden", "tf32_conv_backward_sha256.json")
DEV = "cuda"

# selftest.CONV_SHAPES (B, H, W, Cin, Cout), plus M tails: 33 images leave a partial 128-row tile
SHAPES = [(32, 32, 32, 64, 64), (32, 16, 16, 64, 128), (32, 16, 16, 128, 128), (32, 8, 8, 128, 256),
          (32, 8, 8, 256, 256), (32, 4, 4, 256, 512), (32, 4, 4, 512, 512), (32, 2, 2, 512, 512), (8, 2, 2, 512, 512),
          (8, 32, 32, 64, 64), (33, 8, 8, 128, 128), (33, 2, 2, 512, 512)]
BLOCK_NS = (32, 64, 128, 256)
K_SPLITS = (1, 2, 5, 16)


def cases():
    """(op, shape, block_n, k_split); 0 = the executor's choice."""
    out = []
    for shape in SHAPES:
        cin = shape[3]
        for op in ("dgrad", "wgrad"):
            out.append((op, shape, 0, 0))
            out += [(op, shape, bn, 0) for bn in BLOCK_NS if bn <= cin and cin % bn == 0]
            out += [(op, shape, 0, ks) for ks in K_SPLITS]
    return out


def case_id(c):
    op, (B, H, W, Cin, Cout), bn, ks = c
    return f"{op}-{B}x{H}x{W}-{Cin}-{Cout}-bn{bn}-ks{ks}"


def _inputs(shape):
    B, H, W, Cin, Cout = shape
    g = torch.Generator().manual_seed(B * 1000003 + H * 1009 + Cin * 7 + Cout)      # CPU generator: same inputs anywhere
    x = torch.randn(B, H, W, Cin, generator=g)
    w = torch.randn(Cout, 3, 3, Cin, generator=g) * (1.0 / (9 * Cin) ** 0.5)
    dy = torch.randn(B, H, W, Cout, generator=g)
    return x.to(DEV), w.to(DEV), dy.to(DEV)


def run(N, c, inputs=None):
    """One launch of the case at the executor's defaults for whatever is 0; returns the fp32 result."""
    op, shape, bn, ks = c
    B, H, W, Cin, Cout = shape
    x, w, dy = inputs if inputs is not None else _inputs(shape)
    if op == "dgrad":
        abn, aks = N.conv_tiling(B * H * W, Cin, Cout, flip=1, ke=32)
        tiling = (bn or abn, ks or aks)
        dx = torch.empty(B, H, W, Cin, device=DEV)
        acc = torch.empty(max(1, N.conv_partial_floats(B * H * W, Cin, tiling[1])), device=DEV)
        ctr = torch.zeros(4096, device=DEV, dtype=torch.int32)
        N.conv3x3_dgrad(dy, w, dx, acc=acc, tiling=tiling, counters=ctr)
        torch.cuda.synchronize()
        assert int(ctr.abs().sum()) == 0
        return dx
    dw = torch.zeros(Cout, 3, 3, Cin, device=DEV)
    N.conv3x3_wgrad(x, dy, dw, k_split=ks, block_n=bn)
    torch.cuda.synchronize()
    return dw


def digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def oracle(c, inputs):
    op, shape, _, _ = c
    x, w, dy = (t.double().permute(0, 3, 1, 2) for t in inputs)
    if op == "dgrad":
        return torch.nn.grad.conv2d_input(x.shape, w, dy, padding=1).permute(0, 2, 3, 1)
    return torch.nn.grad.conv2d_weight(x, w.shape, dy, padding=1).permute(0, 2, 3, 1)


def _native():
    from split_learning_b200.ops import native as N
    N.require()
    return N


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.gpu
@pytest.mark.parametrize("c", cases(), ids=case_id)
def test_tf32_backward_bits_and_oracle(c, golden):
    N = _native()
    inputs = _inputs(c[1])
    out = run(N, c, inputs)
    assert digest(out) == golden[case_id(c)], "result bits differ from the recorded kernels"
    ref = oracle(c, inputs)
    err = float((out.double() - ref).abs().max() / ref.abs().max())
    assert err < 4e-3, err
    assert torch.equal(run(N, c, inputs), out), "a repeated launch changed bits"


@pytest.mark.gpu
@pytest.mark.parametrize("shape,tiling", [((32, 2, 2, 512, 512), (64, 16)), ((32, 16, 16, 64, 128), (64, 2)),
                                          ((32, 8, 8, 256, 256), (256, 1))])
def test_tf32_dgrad_publish_graph_replay(shape, tiling):
    """The cut-head dgrad with its mailbox publish, captured in a CUDA graph: every replay gives the eager bits, the
    counters and the ticket come back to zero and the flag is released once per replay."""
    N = _native()
    B, H, W, Cin, Cout = shape
    x, w, dy = _inputs(shape)
    acc = torch.empty(max(1, N.conv_partial_floats(B * H * W, Cin, tiling[1])), device=DEV)
    ctr = torch.zeros(4096, device=DEV, dtype=torch.int32)
    ticket, flag, seq = (torch.zeros(1, device=DEV, dtype=torch.int32) for _ in range(3))
    ref = torch.empty(B, H, W, Cin, device=DEV)
    N.conv3x3_dgrad(dy, w, ref, acc=acc, tiling=tiling, counters=ctr)
    dx = torch.empty_like(ref)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        N.conv3x3_dgrad(dy, w, dx, acc=acc, tiling=tiling, counters=ctr, publish=(ticket, flag, seq))   # warm-up
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        N.conv3x3_dgrad(dy, w, dx, acc=acc, tiling=tiling, counters=ctr, publish=(ticket, flag, seq))
    for i in range(3):
        dx.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(dx, ref)
        assert int(ctr.abs().sum()) == 0 and int(ticket) == 0
        assert int(flag) == int(seq) == i + 2


if __name__ == "__main__":
    if len(sys.argv) != 3 or sys.argv[1] != "--write":
        sys.exit(__doc__)
    N = _native()
    table = {case_id(c): digest(run(N, c)) for c in cases()}
    with open(sys.argv[2], "w") as f:
        json.dump(table, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(table)} digests -> {sys.argv[2]}")
