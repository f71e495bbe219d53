"""Generates the committed golden fixtures tests/golden/*.npz from the fp64 oracle.

PARITY UNPINNED: the reference ships no golden vectors and TensorFlow 1.13.1 cannot be imported here, so
these are OUR pins (regression anchors for the oracle and the CUDA path), not the reference's.
Re-generate with:  python tests/golden/make_golden.py
Inputs are re-created from seeds (SURVEY.md 8d), so the files hold outputs only.
"""
import io
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import tcr_oracle as O  # noqa: E402
from parity_cases import perturbed_variables  # noqa: E402

CASES = {
    "r8_T49": dict(model="TCResNet8", wm=1.0, window=640, stride=320, n=4),
    "r14_T98": dict(model="TCResNet14", wm=1.0, window=480, stride=160, n=3),
}


def save(path, out):
    """Writes `out` as an .npz with LZMA-compressed members.  1-D float32 arrays are stored as their four byte planes
    (uint8 [4, n]): the sign / exponent bytes then compress well, which keeps every fixture under 1 MB."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_LZMA) as z:
        for k, v in out.items():
            v = np.asarray(v)
            if v.dtype == np.float32 and v.ndim == 1:
                v = v.view(np.uint8).reshape(-1, 4).T.copy()
            buf = io.BytesIO()
            np.lib.format.write_array(buf, v)
            z.writestr(k + ".npy", buf.getvalue())


def load(path):
    """Inverse of save() (a plain np.savez file reads the same way): a dict of the stored arrays."""
    gold = np.load(path)
    out = {}
    for k in gold.files:
        v = gold[k]
        out[k] = v.T.copy().view(np.float32).ravel() if v.dtype == np.uint8 else v
    return out


def compute(case):
    t = O.num_frames(16000, case["window"], case["stride"])
    spec = O.build_spec(case["model"], case["wm"], t)
    params, moving = perturbed_variables(spec)
    wav, onehot = O.synthetic_batch(case["n"], adversarial=True)
    feat = O.mfcc(wav, case["window"], case["stride"])
    eval_logits, _ = O.forward(spec, params, moving, feat, False)
    slots = O.zeros_like_vars(spec)
    p1, mv1, s1, ref = O.train_step(spec, params, moving, slots, feat, onehot, 0.1, 0.9, 1e-3)
    out = dict(features=feat.astype(np.float32), eval_logits=eval_logits, train_logits=ref["logits"],
               total_loss=np.float64(ref["total_loss"]), model_loss=np.float64(ref["model_loss"]),
               grads=O.flatten_vars(spec, ref["grads"], np.float64).astype(np.float32),
               params_after=O.flatten_vars(spec, p1, np.float64).astype(np.float32),
               moving_after=O.flatten_moving(spec, mv1, np.float64).astype(np.float32))
    return spec, out


if __name__ == "__main__":
    here = os.path.dirname(os.path.abspath(__file__))
    for name, case in CASES.items():
        _, out = compute(case)
        save(os.path.join(here, name + ".npz"), out)
        print(name, {k: getattr(v, "shape", ()) for k, v in out.items()})
