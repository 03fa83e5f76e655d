"""The ctypes binding declares every C-ABI entry point with the header's types (cutie_b200/kernels.py _SIGNATURES), and the
entry points that take a bank as segments validate its (num_segments, seg_len[]) before any CUDA call.  No GPU needed."""
import ctypes
import os
import re

import pytest

from tests.conftest import ROOT

_SCALARS = {'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'size_t': ctypes.c_size_t, 'float': ctypes.c_float}


def _c_type(decl: str):
    """ctypes type of one C parameter or return type (the name, if any, is dropped)."""
    from cutie_b200.kernels import _QtOp
    if '*' in decl:
        if 'cutie_qt_op' in decl:
            return ctypes.POINTER(_QtOp)
        return ctypes.c_char_p if re.fullmatch(r'const\s+char\s*\*', decl.strip()) else ctypes.c_void_p
    words = decl.split()
    if words == ['void']:
        return None
    base = words[-1] if words[-1] in _SCALARS else words[-2]
    return _SCALARS[base]


def _header_prototypes():
    src = open(os.path.join(ROOT, 'include', 'cutie_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    src = re.sub(r'//[^\n]*', '', src)
    protos = {}
    for ret, name, params in re.findall(r'([A-Za-z_][\w\s]*?\**)\s*\b(cutie_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', src):
        params = ' '.join(params.split())
        args = () if params in ('', 'void') else tuple(_c_type(p) for p in params.split(','))
        assert name not in protos, f'{name} declared twice'
        protos[name] = (_c_type(ret.split('\n')[-1].strip()), args)
    return protos


def test_signature_table_matches_the_header():
    from cutie_b200.kernels import _SIGNATURES
    protos = _header_prototypes()
    assert len(protos) == 50
    assert sorted(_SIGNATURES) == sorted(protos)
    for name, (restype, argtypes) in protos.items():
        got_res, got_args = _SIGNATURES[name]
        assert got_res is restype, (name, got_res, restype)
        assert tuple(got_args) == argtypes, (name, got_args, argtypes)


def test_every_entry_point_the_wrappers_call_is_declared():
    src = open(os.path.join(ROOT, 'cutie_b200', 'kernels.py')).read()
    called = set(re.findall(r"""['"](cutie_[a-z0-9_]+)['"]\s*[,)]""", src)) | set(re.findall(r'\.(cutie_[a-z0-9_]+)\b', src))
    called -= {'cutie_b200'}
    assert len(called) >= 40
    assert called <= set(_header_prototypes()), called - set(_header_prototypes())


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    from cutie_b200 import kernels
    ge.build()
    return kernels.lib()


def test_wrong_python_types_are_rejected_before_the_call(lib):
    for bad in (4096.0, '4096'):
        with pytest.raises(ctypes.ArgumentError):
            lib.cutie_affinity_plan_levels(bad, 30)          # int64_t n_total
        with pytest.raises(ctypes.ArgumentError):
            lib.cutie_set_tc_min_tokens(bad)
    # int64_t in and out: 512 tiles x 256 chunks x 9 taps x 8 KB is more than a C int holds
    assert lib.cutie_conv_weight_image_f16_bytes(1 << 16, 1 << 13, 3) == 512 * 256 * 9 * 8192


_ONE = 0x1000                                                  # never dereferenced: validation fails first


def _arr(ctype, values):
    return (ctype * len(values))(*values)


def _readout_gather(lib, seg_len, K=1):
    ns = len(seg_len)
    return lib.cutie_readout_gather(_ONE, _ONE, 1, 4, 32, ns, _arr(ctypes.c_int64, seg_len),
                                    _arr(ctypes.c_void_p, [_ONE] * (ns * K)), _arr(ctypes.c_int64, [64 * 256] * (ns * K)),
                                    K, 256, _ONE, None)


def test_readout_gather_rejects_a_negative_segment_length_or_five_segments(lib):
    assert _readout_gather(lib, [8, -1]) == -1
    err = lib.cutie_b200_last_error()
    assert b'cutie_readout_gather' in err and b'negative segment length' in err
    assert _readout_gather(lib, [2, 2, 2, 2, 2]) == -1
    err = lib.cutie_b200_last_error()
    assert b'cutie_readout_gather' in err and b'1..4 segments' in err


def test_bank_gather_rejects_a_negative_segment_length(lib):
    st = lib.cutie_bank_gather(2, _arr(ctypes.c_void_p, [_ONE, _ONE]), _arr(ctypes.c_int64, [3, -1]),
                               _arr(ctypes.c_int64, [3 * 64, 64]), _ONE, _ONE, 2 * 64, 1, 2, 64, None)
    assert st == -1
    err = lib.cutie_b200_last_error()
    assert b'cutie_bank_gather' in err and b'negative segment length' in err


def test_consolidation_rejects_a_negative_segment_length_even_when_the_sum_matches(lib):
    P2, I2 = _arr(ctypes.c_void_p, [_ONE, _ONE]), _arr(ctypes.c_int64, [4 * 64, 64])
    st = lib.cutie_consolidate_partial(2, P2, P2, _arr(ctypes.c_int64, [4, -1]), I2, I2, P2, I2, 1, _ONE, 64, _ONE, 64,
                                       1, 1, 64, 256, _arr(ctypes.c_void_p, [_ONE]), _arr(ctypes.c_int64, [256]), _ONE, 1,
                                       None, None, _ONE, 3, None)
    assert st == -1
    err = lib.cutie_b200_last_error()
    assert b'cutie_consolidate_partial' in err and b'negative segment length' in err
