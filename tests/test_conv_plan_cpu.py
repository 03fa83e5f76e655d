"""Host logic of cutie_conv_tc's launch plan (csrc/conv_tc.cu, no GPU needed: cutie_conv_plan is arithmetic only): the
(output tile, input chunk) unit ranges handed to the CTAs, restated here the way the kernel decodes them -- every unit is
computed exactly once, a CTA's share spans at most two tiles, the shares of a tile carry the slots 0 .. n-1 and fit the
workspace, layers smaller than the GPU are spread over (at most) all SMs."""
import ctypes

import pytest

SMS = 132                      # num_sms() falls back to 132 without a device (H100 SXM)


def _plan(K_, NB, Cin, Cout, H, W, k, s, q=0):
    out = (ctypes.c_int64 * 6)()
    st = K_.lib().cutie_conv_plan(ctypes.c_int64(NB), ctypes.c_int64(Cin), ctypes.c_int64(Cout), ctypes.c_int64(H),
                                  ctypes.c_int64(W), k, s, q, out)
    assert st == 0, K_.lib().cutie_b200_last_error()
    return tuple(out)          # T, N, C, q, CTAs, workspace floats


def _shares(T, C, q, ctas):
    """The kernel's decoding of blockIdx.x -> [(tile, c0, c1, slot, nslots)] (conv_tc_kernel::make_part)."""
    U = T * C
    for i in range(ctas):
        u0, u1 = i * q, min(U, i * q + q)
        split_at = min((u0 // C + 1) * C, u1)
        parts = [(u0, split_at)] + ([(split_at, u1)] if split_at < u1 else [])
        out = []
        for ua, ub in parts:
            t = ua // C
            first, last = (t * C) // q, (t * C + C - 1) // q
            out.append((t, ua - t * C, ua - t * C + (ub - ua), i - first, last - first + 1))
        yield out


LAYERS = [(3, 256, 256, 30, 54, 3, 1), (1, 256, 256, 30, 54, 3, 1), (1, 1024, 256, 30, 54, 1, 1), (1, 256, 1024, 30, 54, 1, 1),
          (1, 64, 256, 120, 216, 1, 1), (3, 128, 128, 120, 216, 3, 1), (3, 512, 768, 30, 54, 3, 1), (1, 128, 128, 120, 216, 3, 2),
          (3, 128, 256, 60, 108, 3, 2), (1, 512, 1024, 60, 108, 1, 2), (2, 96, 200, 7, 9, 3, 1), (1, 32, 64, 3, 5, 1, 1),
          (1, 64, 128, 1, 1, 3, 1), (15, 256, 256, 30, 54, 3, 1)]


@pytest.mark.parametrize('NB,Cin,Cout,H,W,k,s', LAYERS)
@pytest.mark.parametrize('q_override', [0, 1, 2, 3, 5, 7])
def test_every_unit_is_computed_once_and_slots_are_dense(NB, Cin, Cout, H, W, k, s, q_override):
    import cutie_b200.kernels as K_
    T, N, C, q, ctas, ws = _plan(K_, NB, Cin, Cout, H, W, k, s, q_override)
    assert C == Cin // 32 and 1 <= q <= C and 16 <= N <= 128 and N % 16 == 0
    assert ctas == -(-T * C // q)
    if q_override == 0:
        assert C % q == 0 and (q == C or (ctas <= SMS and q >= 2))     # uniform splits only, never more CTAs than SMs
    assert (ws == 0) == (q >= C)
    maxslots = ws // (T * N * 128) if ws else 1
    seen = {}
    slots = {}
    for share in _shares(T, C, q, ctas):
        assert 1 <= len(share) <= 2
        for t, c0, c1, slot, nslots in share:
            assert 0 <= t < T and 0 <= c0 < c1 <= C and 0 <= slot < nslots <= maxslots
            for c in range(c0, c1):
                assert (t, c) not in seen
                seen[(t, c)] = True
            slots.setdefault(t, []).append((slot, nslots))
    assert len(seen) == T * C
    for t, ss in slots.items():
        assert sorted(s_ for s_, _ in ss) == list(range(len(ss))) and all(n == len(ss) for _, n in ss)


@pytest.mark.parametrize('H,W', [(30, 54), (60, 108), (120, 216), (17, 130), (1, 1), (5, 7), (23, 40), (270, 480)])
def test_3x3_tile_shape_fits_the_activation_stage(H, W):
    import cutie_b200.kernels as K_
    out = (ctypes.c_int * 3)()
    assert K_.lib().cutie_debug_conv_tile_shape(ctypes.c_int64(H), ctypes.c_int64(W), out) == 0
    th, tw, n = tuple(out)
    assert th >= 1 and tw >= 1 and n % 16 == 0 and th * (tw + 2) <= n <= 128
    assert n + 2 * (tw + 2) + 2 <= 248                       # rows of the local padded grid + slack (CV3_ROWS)


def test_3x3_boundary_widths_of_the_gpu_tests_straddle_a_tile_shape_change():
    """tests/test_gpu_conv_tc.py runs 30 x 57 and 30 x 58 to cover both sides of a change of tile shape: one whole-row
    column tile per row, then two column tiles."""
    import cutie_b200.kernels as K_
    out = (ctypes.c_int * 3)()
    shapes = []
    for W in (57, 58):
        assert K_.lib().cutie_debug_conv_tile_shape(ctypes.c_int64(30), ctypes.c_int64(W), out) == 0
        shapes.append(tuple(out))
    assert shapes[0][1] == 57 and shapes[1][1] < 58, shapes
