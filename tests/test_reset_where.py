"""Device-side resets (cassie_batch_reset_where, and the masked cassie_batch_set_state that runs the same kernel): the product's restore source
(csrc/reset.inl) in the host emulation, against a numpy gather of random rows, and the C-ABI / Python surface of the four verbs.  The GPU tests are in
tests/test_gpu_reset_where.py.

The emulation is tests/emu/emu_reset.cpp, built into its own library here.  Rows are random bytes: the restore is a bitwise copy, the same in both
precisions except for the row widths."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import REPO

RR = ['qpos', 'qvel', 'qacc', 'cst', 'xfrc', 'obs', 'dfilt', 'est', 'aux', 'applied', 'frames', 'acc']   # reset.inl RR_* order
OPTIONAL = {'est', 'aux', 'applied', 'frames', 'acc'}
NFR = 3
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_reset.so')
        srcs = [os.path.join(E.HERE, 'emu', 'emu_reset.cpp')] + [os.path.join(E.CSRC, f) for f in ('reset.inl', 'step_core.inl', 'devmodel.h', 'estimator_host.h')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0]])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, ci = C.c_void_p, C.c_int
        L.emu_reset_bytes.argtypes = [ci, ci, ci, ci, C.POINTER(ci)]
        L.emu_reset.argtypes = [C.POINTER(vp), C.POINTER(vp), ci, ci, ci, ci, ci, vp, vp, ci, ci]
        _LIB = L
    return _LIB


def row_bytes(esz, qw, vw, nframes=NFR):
    b = (C.c_int * len(RR))()
    assert lib().emu_reset_bytes(esz, qw, vw, nframes, b) == len(RR)
    return dict(zip(RR, b))


def run(dst, src, esz, qw, vw, mask, entry, k, n, same_frames=True):
    """dst / src: dict kind -> uint8 [rows, bytes] (a missing kind: the batch / bank lacks it); dst is restored in place"""
    keep = []
    d = (C.c_void_p * len(RR))(*[dst[r].ctypes.data if r in dst else None for r in RR])
    s = (C.c_void_p * len(RR))(*[src[r].ctypes.data if r in src else None for r in RR])
    if mask is not None:
        mask = np.ascontiguousarray(mask, dtype=np.uint8); keep.append(mask)
    if entry is not None:
        entry = np.ascontiguousarray(entry, dtype=np.int32); keep.append(entry)
    return lib().emu_reset(d, s, esz, qw, vw, NFR, 1 if same_frames else 0, None if mask is None else mask.ctypes.data,
                           None if entry is None else entry.ctypes.data, k, n)


def rows(rng, kinds, bytes_, count):
    return {r: rng.integers(0, 256, size=(count, bytes_[r]), dtype=np.uint8) for r in kinds}


def expected(dst, src, mask, entry, k, n, same_frames=True):
    """the numpy gather by the rules of cassie_batch_reset_where"""
    idx = (np.arange(n, dtype=np.uint32) if entry is None else np.asarray(entry, dtype=np.int32).view(np.uint32)) % np.uint32(k)
    sel = np.ones(n, bool) if mask is None else np.asarray(mask) != 0
    out = {r: v.copy() for r, v in dst.items()}
    for r, v in out.items():
        if r in ('est', 'applied') and r not in src:
            v[sel] = 0                                      # zeroed: the filters start afresh, no force acts
        elif r in src and (same_frames or r not in ('frames', 'acc')):
            v[sel] = src[r][idx[sel]]
    return out


WIDTHS = [(4, 36, 32), (4, 44, 40), (8, 36, 32), (8, 44, 40)]   # fp32 / fp64, cassie.xml / cassie_tray_box.xml (the extra free body)


def test_every_row_is_a_whole_number_of_16_byte_words():
    for esz, qw, vw in WIDTHS:
        for nfr in (0, 1, 8, 64):
            b = row_bytes(esz, qw, vw, nfr)
            assert all(v % 16 == 0 for v in b.values()), (esz, qw, b)
    b = row_bytes(4, 36, 32, 8)
    assert (b['qpos'], b['qvel'], b['cst'], b['xfrc'], b['obs'], b['dfilt'], b['est'], b['aux'], b['applied'], b['frames'], b['acc']) == \
        (144, 128, 768, 32, 448, 384, 1024, 256, 928, 640, 416)


@pytest.mark.parametrize('esz,qw,vw', WIDTHS)
def test_restore_equals_the_numpy_gather(esz, qw, vw):
    rng = np.random.default_rng(esz * 100 + qw)
    b = row_bytes(esz, qw, vw)
    for n, k in ((257, 64), (64, 1), (40, 300)):
        dst, src = rows(rng, RR, b, n), rows(rng, RR, b, k)
        mask = (rng.random(n) < 0.3).astype(np.uint8) * rng.integers(1, 256, n).astype(np.uint8)   # any non-zero byte selects
        entry = rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(np.int32)
        entry[:8] = [-1, -k, k, k + 1, 2 ** 31 - 1, -2 ** 31, 0, k - 1]
        want = expected(dst, src, mask, entry, k, n)
        assert run(dst, src, esz, qw, vw, mask, entry, k, n) == int((mask != 0).sum())
        for r in RR:
            assert np.array_equal(dst[r], want[r]), r


@pytest.mark.parametrize('esz,qw,vw', WIDTHS)
def test_null_entry_takes_e_mod_k_and_null_mask_takes_all(esz, qw, vw):
    rng = np.random.default_rng(7)
    b = row_bytes(esz, qw, vw)
    n, k = 100, 7
    dst, src = rows(rng, RR, b, n), rows(rng, RR, b, k)
    want = expected(dst, src, None, None, k, n)
    assert run(dst, src, esz, qw, vw, None, None, k, n) == n
    for r in RR:
        assert np.array_equal(dst[r], want[r]), r
        assert np.array_equal(dst[r], src[r][np.arange(n) % k]), r


@pytest.mark.parametrize('esz,qw,vw', WIDTHS)
@pytest.mark.parametrize('lacking', ['est', 'applied', 'aux', 'frames', 'acc'])
def test_a_row_kind_the_bank_lacks(esz, qw, vw, lacking):
    """est and applied rows are zeroed for the restored environments, aux, frame and acceleration rows left alone; unmasked rows never change"""
    rng = np.random.default_rng(11)
    b = row_bytes(esz, qw, vw)
    n, k = 96, 16
    dst, src = rows(rng, RR, b, n), rows(rng, [r for r in RR if r != lacking], b, k)
    before = {r: v.copy() for r, v in dst.items()}
    mask = (rng.random(n) < 0.5).astype(np.uint8)
    entry = rng.integers(-50, 50, n).astype(np.int32)
    run(dst, src, esz, qw, vw, mask, entry, k, n)
    sel = mask != 0
    if lacking in ('est', 'applied'):
        assert not dst[lacking][sel].any()
    else:
        assert np.array_equal(dst[lacking], before[lacking])
    for r in RR:
        assert np.array_equal(dst[r][~sel], before[r][~sel]), r
    assert np.array_equal(dst['qpos'][sel], src['qpos'][(entry[sel].view(np.uint32) % k)])


@pytest.mark.parametrize('esz,qw,vw', WIDTHS)
def test_other_frame_list_leaves_frames_and_acc_alone(esz, qw, vw):
    rng = np.random.default_rng(13)
    b = row_bytes(esz, qw, vw)
    n, k = 50, 9
    dst, src = rows(rng, RR, b, n), rows(rng, RR, b, k)
    mask = np.ones(n, np.uint8)
    entry = rng.integers(0, 1000, n).astype(np.int32)
    want = expected(dst, src, mask, entry, k, n, same_frames=False)
    run(dst, src, esz, qw, vw, mask, entry, k, n, same_frames=False)
    for r in RR:
        assert np.array_equal(dst[r], want[r]), r
    assert np.array_equal(dst['aux'], src['aux'][entry.view(np.uint32) % k])


@pytest.mark.parametrize('esz,qw,vw', WIDTHS)
def test_a_row_kind_the_batch_lacks_is_ignored(esz, qw, vw):
    rng = np.random.default_rng(17)
    b = row_bytes(esz, qw, vw)
    n, k = 40, 5
    have = [r for r in RR if r not in OPTIONAL]
    dst, src = rows(rng, have, b, n), rows(rng, RR, b, k)
    mask = (rng.random(n) < 0.5).astype(np.uint8)
    want = expected(dst, src, mask, None, k, n)
    run(dst, src, esz, qw, vw, mask, None, k, n)
    for r in have:
        assert np.array_equal(dst[r], want[r]), r


# ---- the C-ABI and the Python surface

VERBS = ['cassie_batch_set_reset_bank', 'cassie_batch_reset_bank_size', 'cassie_batch_reset_where', 'cassie_batch_forward_where']


def test_verbs_are_declared_and_exported(pkg):
    hdr = re.sub(r'/\*.*?\*/', '', open(os.path.join(REPO, 'include', 'cassie_b200.h')).read(), flags=re.S)
    for v in VERBS:
        assert re.search(r'\bint\s+%s\s*\(' % v, hdr), v
    pkg.build()
    L = C.CDLL(pkg.LIB_PATH)
    for v in VERBS:
        assert hasattr(L, v), v


def test_ctypes_wrappers_set_argtypes_and_restypes(pkg):
    b = object.__new__(pkg.CassieBatch)
    b.L = pkg.lib()
    L = b._reset_lib()
    vp = C.c_void_p
    assert L.cassie_batch_set_reset_bank.argtypes == [vp, vp, C.POINTER(C.c_int), C.c_int]
    assert L.cassie_batch_reset_bank_size.argtypes == [vp]
    assert L.cassie_batch_reset_where.argtypes == [vp, vp, vp]
    assert L.cassie_batch_forward_where.argtypes == [vp, vp]
    for v in VERBS:
        assert getattr(L, v).restype is C.c_int, v


def test_python_refuses_host_masks_before_the_library_is_called(pkg):
    torch = pytest.importorskip('torch')
    b = object.__new__(pkg.CassieBatch)
    b.L, b.n, b.device, b.h = pkg.lib(), 4, 0, None   # h None: a call that reached the library would fail differently
    for bad in (np.ones(4, np.uint8), torch.ones(4, dtype=torch.bool), [1, 0, 1, 0]):
        with pytest.raises((TypeError, ValueError)):
            b.reset_where(bad)
        with pytest.raises((TypeError, ValueError)):
            b.forward_where(bad)
