"""Generates tests/golden/e2e_many_objects.npz by running the UNMODIFIED reference on CPU.

Run from the repository root where the reference is installed (oracle/_ref/, made by __graft_entry__.build(); or
CUTIE_REFERENCE_ROOT):
    python tests/golden/make_golden_many_objects.py

e2e_many_objects.npz  free-running InferenceCore.step with 20 objects in one bucket (FIFO memory, 96x160): segment()
                      logits per frame and the memory size trace.  20 objects is past the 16 objects one launch of the
                      readout gather and consolidation kernels takes, so the fixture pins their grouped launches.
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
warnings.filterwarnings('ignore')

from make_golden import OUT, rh, run_e2e      # noqa: E402  (also puts the repository root on sys.path)

T, H, W, K = 8, 96, 160, 20
CFG = dict(mem_every=2, max_mem_frames=3)
STRIDE = 8          # logits and probabilities are kept at every 8th row and column (full planes would be 9 MB)


def main():
    ref = rh.load_reference()
    net = rh.build_reference_model(rh.reference_cfg())
    run_e2e(ref, net, rh.reference_cfg(**CFG), 'many_objects', T=T, H=H, W=W, K=K)
    path = os.path.join(OUT, 'e2e_many_objects.npz')
    rec = dict(np.load(path))
    rec['logits'] = np.ascontiguousarray(rec['logits'][:, :, ::STRIDE, ::STRIDE])
    rec['final_prob'] = np.ascontiguousarray(rec['final_prob'][:, ::STRIDE, ::STRIDE])
    rec['logits_stride'] = np.array(STRIDE)
    del rec['masks']
    np.savez_compressed(path, **rec)


if __name__ == '__main__':
    main()
