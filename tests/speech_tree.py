"""A small Speech Commands directory tree for the loader tests: seeded clips of several lengths and sample types per class,
``testing_list.txt`` / ``validation_list.txt`` holding some of them out of the training split, one truncated (unreadable)
file and one int16 stereo file."""
import os

import numpy as np

from split_learning_b200.data.speechcommands import CLASSES, SAMPLE_RATE

L = 15920


def clip(rng, kind: int, n: int) -> np.ndarray:
    t = np.arange(n) / SAMPLE_RATE
    if kind == 0:                                           # int16 tone
        return (np.sin(2 * np.pi * rng.uniform(200, 4000) * t) * rng.uniform(2000, 30000)).astype(np.int16)
    if kind == 1:                                           # float32 noise
        return (rng.standard_normal(n) * 0.05).astype(np.float32)
    return (rng.standard_normal(n) * 3000).clip(-32768, 32767).astype(np.int16)     # int16 noise


def make_tree(root, per_class: int = 3, seed: int = 0) -> dict:
    """Writes ``per_class`` training clips per class plus held-out ones; returns {"train": [(relpath, label)],
    "unreadable": relpath, "stereo": relpath}."""
    from scipy.io import wavfile
    rng = np.random.default_rng(seed)
    base = os.path.join(str(root), "SpeechCommands", "speech_commands_v0.02")
    train, held_test, held_val = [], [], []
    for ci, c in enumerate(CLASSES):
        os.makedirs(os.path.join(base, c), exist_ok=True)
        for j in range(per_class + 2):
            name = f"{c}/clip{j:03d}.wav"
            n = [L, 8000, 20000, L - 7, 16000][(ci + j) % 5]
            wavfile.write(os.path.join(base, name), SAMPLE_RATE, clip(rng, (ci + j) % 3, n))
            if j == per_class:
                held_test.append(name)
            elif j == per_class + 1:
                held_val.append(name)
            else:
                train.append((name, ci))
    stereo = "left/stereo.wav"
    wavfile.write(os.path.join(base, stereo), SAMPLE_RATE, np.stack([clip(rng, 0, 9000), clip(rng, 2, 9000)], axis=1))
    train.append((stereo, CLASSES.index("left")))
    bad = "go/broken.wav"
    wavfile.write(os.path.join(base, bad), SAMPLE_RATE, clip(rng, 0, L))
    with open(os.path.join(base, bad), "r+b") as f:
        f.truncate(30)
    train.append((bad, CLASSES.index("go")))
    with open(os.path.join(base, "testing_list.txt"), "w") as f:
        f.write("\n".join(held_test) + "\n")
    with open(os.path.join(base, "validation_list.txt"), "w") as f:
        f.write("\n".join(held_val) + "\n")
    return {"train": train, "unreadable": bad, "stereo": stereo, "base": base}
