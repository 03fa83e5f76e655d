"""frame_graphs._Captured pauses Python's cyclic garbage collector while a CUDA graph is being captured: the collector can
run at any allocation, and finalising a dead reference cycle that holds another captured graph (a discarded
InferenceCore -- its encoder look-ahead refers back to it) destroys that graph and releases its memory pool in the middle
of the capture, which invalidates the capture.  Driven on the CPU with stand-ins for the torch.cuda graph and stream API."""
import contextlib
import gc

import torch


class _Stream:
    def wait_stream(self, other):
        pass


def _stand_ins(monkeypatch, seen):
    class _Graph:
        def replay(self):
            pass

    @contextlib.contextmanager
    def graph(g):
        seen.append(('capture', gc.isenabled()))
        yield
    monkeypatch.setattr(torch.cuda, 'CUDAGraph', _Graph)
    monkeypatch.setattr(torch.cuda, 'graph', graph)
    monkeypatch.setattr(torch.cuda, 'Stream', _Stream)
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: _Stream())
    monkeypatch.setattr(torch.cuda, 'stream', lambda s: contextlib.nullcontext())


def test_capture_runs_with_the_cyclic_collector_paused(monkeypatch):
    from cutie_b200.inference import frame_graphs as fg
    seen = []
    _stand_ins(monkeypatch, seen)

    def fn(x):
        seen.append(('fn', gc.isenabled()))
        return x + 1
    assert gc.isenabled()
    cap = fg._Captured(fn, (torch.zeros(2),))
    assert seen == [('fn', True), ('fn', True), ('capture', False), ('fn', False)]    # warm-up runs, then the capture
    assert gc.isenabled() and torch.equal(cap.outputs, torch.ones(2))


def test_collector_is_restored_when_the_capture_fails(monkeypatch):
    from cutie_b200.inference import frame_graphs as fg
    seen = []
    _stand_ins(monkeypatch, seen)
    calls = []

    def fn(x):
        calls.append(1)
        if len(calls) == 3:
            raise RuntimeError('capture failed')
        return x
    try:
        fg._Captured(fn, (torch.zeros(1),))
    except RuntimeError:
        pass
    assert gc.isenabled()
    gc.disable()                                          # a caller that had it off keeps it off
    try:
        fg._Captured(lambda x: x, (torch.zeros(1),))
        assert not gc.isenabled()
    finally:
        gc.enable()
