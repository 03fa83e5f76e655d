"""The UNMODIFIED reference (oracle/_ref/) run as tests/ref_runner.py runs it, except that every `InferenceCore.step` is
called inside torch.autocast('cuda', dtype=torch.float16) -- what the reference's own drivers do (scripting_demo.py:13
`@torch.cuda.amp.autocast()`, cutie/eval_vos.py:112 with `amp: True`).  Same child, same job format and result dict as
tests/ref_runner.py; only the step is wrapped.

TEST INFRASTRUCTURE ONLY.  Parent side: `run_reference_clip_amp(...)`; child side: `python tests/ref_runner_amp.py in.pt out.pt`.
"""
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import ref_runner  # noqa: E402


def run_reference_clip_amp(frames, mask, objects, *, device='cuda', cfg_overrides=None, max_internal_size=-1,
                           snapshot=False, timeout=900):
    """frames: list of [3,H,W] float CPU tensors; mask: index mask [H,W]; returns ref_runner's result dict (logits of the
    propagated frames as fp32, output masks) for the reference under fp16 autocast."""
    root = ref_runner.reference_root()
    if root is None:
        raise RuntimeError('no reference tree (oracle/_ref missing: run `python oracle/install_reference.py`)')
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, 'in.pt'), os.path.join(tmp, 'out.pt')
        torch.save(dict(frames=[f.cpu() for f in frames], mask=mask.cpu(), objects=list(objects), device=device,
                        cfg_overrides=dict(cfg_overrides or {}), max_internal_size=max_internal_size,
                        snapshot=snapshot, exact_similarity=False), fin)
        env = dict(os.environ, CUTIE_REFERENCE_ROOT=root)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), fin, fout], env=env, cwd=ROOT,
                           capture_output=True, text=True, timeout=timeout)
        if r.returncode != 0:
            raise RuntimeError('reference child failed:\n' + r.stdout[-2000:] + '\n' + r.stderr[-4000:])
        return torch.load(fout, weights_only=False)


def _child_amp(fin, fout):
    from oracle import ref_harness as rh
    load = rh.load_reference

    def load_with_autocast_step():
        ref = load()
        cls = ref.InferenceCore
        if not getattr(cls, '_step_under_autocast', False):
            step = cls.step

            def step_under_autocast(self, *a, **kw):
                with torch.autocast('cuda', dtype=torch.float16):
                    return step(self, *a, **kw)
            cls.step = step_under_autocast
            cls._step_under_autocast = True
        return ref
    rh.load_reference = load_with_autocast_step      # ref_runner's child loads the reference through this name
    ref_runner._child(fin, fout)


if __name__ == '__main__':
    _child_amp(sys.argv[1], sys.argv[2])
