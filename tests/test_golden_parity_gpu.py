"""Golden parity (SURVEY §4): the UNMODIFIED reference trainers (the reference's ``src/train/VGG16.py`` first-layer and
last-layer loops, reference model classes, torch SGD over an in-process pika shim) ran 20 microbatches of VGG16 / CIFAR10 cut
at layer 7 — once as shipped (cuDNN's default TF32 convolutions) and once with ``torch.backends.cudnn.allow_tf32 = False``
(exact fp32, the oracle).  ``tools/make_golden.py`` stored their losses, the same fixed random sample of every cut activation
and cut gradient, and samples of seven final weight tensors in ``tests/golden/parity_vgg16_cut7.npz``.  The native engine in
its default precision (wgmma tf32 convolutions, fp32 Linear / BN / SGD) runs the same 20 microbatches from the same initial
weights.  Per step: training loss, the activation that crosses the cut, the gradient that comes back.

Criterion: the native engine must be as close to the fp32 oracle as the reference's own TF32 run is (a random-init VGG on
noise amplifies operand rounding through ReLU / max-pool decision flips: the reference-TF32 cut gradient itself sits at
cos ~0.96-0.99 against the oracle, so a fixed "cos > 0.999" would fail the reference against itself), and match the
reference-TF32 loss trajectory to well under 1 %.  Dropout is switched off in both (its random streams cannot match);
control-count 1 makes the forward / backward interleaving deterministic in both engines."""
import numpy as np
import pytest
import torch

from oracle_cases import PARITY_KEYS, PARITY_LEARNING, STEPS, B, golden_path, parity_batches, parity_initial_stages

pytestmark = pytest.mark.gpu


def test_golden_parity_vs_reference_trainers():
    from split_learning_b200.models import VGG16_CIFAR10
    from split_learning_b200.ops import native as N
    from split_learning_b200.parallel.pipeline import LocalPipeline
    from split_learning_b200.train.b200_executor import B200Executor
    N.require()
    dev = torch.device("cuda:0")
    gold = np.load(golden_path("parity_vgg16_cut7.npz"))
    batches = parity_batches()
    ref_loss, ex_loss = gold["loss_tf32"].tolist(), gold["loss_fp32"].tolist()
    ref_act, ex_act, ref_grad, ex_grad = gold["act_tf32"], gold["act_fp32"], gold["grad_tf32"], gold["grad_fp32"]
    assert len(ref_loss) == STEPS and len(ref_act) == STEPS and len(ref_grad) == STEPS and len(ex_loss) == STEPS
    act_idx = torch.from_numpy(gold["act_idx"]).to(dev)
    grad_idx = torch.from_numpy(gold["grad_idx"]).to(dev)

    learning = dict(PARITY_LEARNING, precision="tf32")
    m1, m2 = parity_initial_stages(VGG16_CIFAR10)          # the reference run's initial weights
    base = {k: v.detach().clone().float().flatten() for k, v in list(m1.state_dict().items()) + list(m2.state_dict().items())}
    ex1 = B200Executor(m1, "VGG16", learning, dev, is_first=True)
    ex2 = B200Executor(m2, "VGG16", learning, dev, is_last=True)
    for b in ex2.blocks:                                   # dropout off, like the recorded reference run
        if hasattr(b, "drop"):
            b.drop = 0.0
        if hasattr(b, "p"):
            b.p = 0.0
    pipe = LocalPipeline([ex1, ex2], B, 1)
    act_mb, grad_mb = pipe.stages[0].fwd_out, pipe.stages[0].grad_in
    loss, acts, grads = [], [], []
    for x, y in batches:
        if pipe.it_f - pipe.it_b >= pipe.depth:
            pipe.step_backward()
        pipe.feed(x.pin_memory(), y.pin_memory())
        pipe.step_forward()
        pipe.synchronize()
        loss.append(float(pipe.loss()[0]))
        acts.append(act_mb.payload[0].float().permute(0, 3, 1, 2).flatten()[act_idx].cpu().numpy())   # NHWC slot -> NCHW
        grads.append(grad_mb.payload[0].float().permute(0, 3, 1, 2).flatten()[grad_idx].cpu().numpy())
    while pipe.it_b < pipe.it_f:
        pipe.step_backward()
    pipe.synchronize()

    # over the stored samples of each tensor
    cosf = lambda a, b: float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b)))
    relf = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())

    def deviation(L, A, G):
        """worst-over-steps deviation of a run from the fp32 oracle"""
        return (max(abs(a - b) / abs(b) for a, b in zip(L, ex_loss)), max(relf(a, b) for a, b in zip(A, ex_act)),
                max(1.0 - cosf(a, b) for a, b in zip(G, ex_grad)))
    ours, theirs = deviation(loss, acts, grads), deviation(ref_loss, ref_act, ref_grad)
    worst_loss = max(abs(a - b) / abs(b) for a, b in zip(loss, ref_loss))
    print(f"golden parity over {STEPS} steps — deviation from the fp32 oracle (loss rel, cut activation rel, cut gradient 1-cos): "
          f"native {ours[0]:.2e} {ours[1]:.2e} {ours[2]:.2e} | reference TF32 {theirs[0]:.2e} {theirs[1]:.2e} {theirs[2]:.2e}; "
          f"native vs reference-TF32 loss rel {worst_loss:.2e}; step-0 gradient cos native {cosf(grads[0], ex_grad[0]):.5f} "
          f"reference {cosf(ref_grad[0], ex_grad[0]):.5f}")
    assert worst_loss < 5e-3, (loss, ref_loss)                       # loss trajectory within 0.5 % of the reference as shipped
    assert ours[0] < 2 * theirs[0] + 2e-4, (ours, theirs)
    assert ours[1] < 2 * theirs[1] + 5e-4, (ours, theirs)
    assert ours[2] < 2 * theirs[2] + 2e-3, (ours, theirs)
    assert relf(acts[0], ex_act[0]) < 1e-3                           # step 0 (identical weights): plain TF32 operand rounding
    # final weights: the engines took the same 20 SGD steps — compare against the oracle, relative to how far it moved
    out1, out2 = ex1.state_dict(), ex2.state_dict()
    for k in PARITY_KEYS:
        idx = torch.from_numpy(gold[f"{k}:idx"])
        mine = (out1 if k in out1 else out2)[k].float().cpu().flatten()[idx].numpy()
        start = base[k].cpu()[idx].numpy()
        oracle, ref = gold[f"{k}:fp32"], gold[f"{k}:tf32"]
        moved = float(np.abs(oracle - start).max())
        e_mine, e_ref = float(np.abs(mine - oracle).max()), float(np.abs(ref - oracle).max())
        print(f"  final {k}: oracle moved {moved:.3e}; off the oracle: native {e_mine:.3e}, reference TF32 {e_ref:.3e}")
        assert moved > 0 and e_mine < 2 * e_ref + 0.02 * moved + 1e-7, (k, moved, e_mine, e_ref)
    nbt = int(out1["layer2.num_batches_tracked"])
    assert nbt == int(gold["nbt"]) == 2 * STEPS                      # forward + recompute, as in the reference
