"""GPU checks of the typed VF-vGPU CDI layouts (additions to ABI v14): kxpu_cdi_emit_vf_vgpu[_cdev] is bit-exact against
the C oracle (tests/vf_vgpu_cdi_oracle.c) for both formats, 3-, 14- and 63-byte kinds and 0 .. 2^20 devices, and
kxpu_cdi_parse_vf_vgpu[_cdev] gives the records back for each of those documents; the six CDI layouts refuse each
other's documents; every domain violation is KXPU_E_UNSUPPORTED with nothing written; the two-call sizing and the
KXPU_E_NOSPACE protocol behave as for the other layouts."""
import ctypes as C

import numpy as np
import pytest

import cdi_parse_cases as CP
import mdev_cdev_cases as MC
import vf_vgpu_cdi_cases as K
import vf_vgpu_cdi_oracle as VO
from kxpu_b200 import binding as B

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 127, 128, 129, 65536, 1 << 20]


def _emit_raw(kx, cdev):
    return kx.L.kxpu_cdi_emit_vf_vgpu_cdev if cdev else kx.L.kxpu_cdi_emit_vf_vgpu


@pytest.mark.parametrize("cdev", [False, True])
@pytest.mark.parametrize("kind", K.KINDS)
@pytest.mark.parametrize("fmt", [K.FMT_YAML, K.FMT_JSON])
@pytest.mark.parametrize("n", SIZES)
def test_emit_and_parse(kx, n, fmt, kind, cdev):
    recs = K.records(n, seed=n + 13)
    want = VO.emit(fmt, kind, recs, cdev)
    got = kx.cdi_emit_vf_vgpu(fmt, recs, kind, cdev=cdev)
    assert got == want
    back = kx.cdi_parse_vf_vgpu(fmt, got, kind, cdev=cdev)
    assert len(back) == n
    assert back.tobytes() == (recs if cdev else K.group_view(recs)).tobytes()
    if 0 < n <= 129:  # the host buffer at every 16-byte phase
        for off in range(16):
            rc, m, out = kx.cdi_parse_raw(fmt, got, kind, n, offset=off, cdev=cdev, typed=True)
            assert (rc, m) == (B.KXPU_OK, n), off
            assert out.tobytes() == back.tobytes(), off


@pytest.mark.parametrize("fmt", [K.FMT_YAML, K.FMT_JSON])
def test_layouts_refuse_each_other(kx, fmt):
    kind = K.KIND_14
    recs = K.records(300, seed=8)
    mrecs = MC.records(300, seed=8)
    docs = {"kind": kx.cdi_emit(fmt, recs["dev"], kind), "cdev": kx.cdi_emit_cdev(fmt, recs["dev"], kind),
            "mdev": kx.cdi_emit_mdev(fmt, mrecs["dev"], kind), "mdev_cdev": kx.cdi_emit_mdev_cdev(fmt, mrecs, kind),
            "typed": kx.cdi_emit_vf_vgpu(fmt, recs, kind), "typed_cdev": kx.cdi_emit_vf_vgpu(fmt, recs, kind, cdev=True)}
    parsers = {"kind": dict(), "cdev": dict(cdev=True), "mdev": dict(mdev=True), "mdev_cdev": dict(mdev=True, cdev=True),
               "typed": dict(typed=True), "typed_cdev": dict(typed=True, cdev=True)}
    for dname, doc in docs.items():
        for pname, how in parsers.items():
            rc, n, _ = kx.cdi_parse_raw(fmt, doc, kind, 300, **how)
            assert rc == (B.KXPU_OK if dname == pname else B.E_INVALID), (dname, pname)
            assert n == (300 if dname == pname else -1), (dname, pname)
    # the zero-device document is the same bytes in every layout, and every parser reads it as no device
    zero = kx.cdi_emit_vf_vgpu(fmt, recs[:0], kind)
    assert zero == kx.cdi_emit_vf_vgpu(fmt, recs[:0], kind, cdev=True) == kx.cdi_emit(fmt, recs["dev"][:0], kind)
    assert zero == kx.cdi_emit_mdev_cdev(fmt, mrecs[:0], kind)
    for how in parsers.values():
        assert kx.cdi_parse_raw(fmt, zero, kind, 0, **how)[:2] == (B.KXPU_OK, 0)


@pytest.mark.parametrize("cdev", [False, True])
def test_domain_violations_write_nothing(kx, cdev):
    good = K.records(200, seed=5)
    bad = []
    r = good.copy(); r["type_id"][150] = 0; bad.append(r)
    r = good.copy(); r["key_len"][150] = 0; bad.append(r)
    r = good.copy(); r["key_len"][150] = 41; bad.append(r)
    for c in (b" ", b"/", b'"', b":", b"\xff", b"\x00", b"\\"):
        r = good.copy(); key = bytearray(b"abcdefgh".ljust(40, b"\0")); key[5:6] = c
        r["key"][150] = bytes(key); r["key_len"][150] = 8; bad.append(r)
    r = good.copy(); r["dev"]["bdf"][150] = b"0000:C1:00.0"; bad.append(r)
    fn = _emit_raw(kx, cdev)
    for fmt in (K.FMT_YAML, K.FMT_JSON):
        for k, r in enumerate(bad):
            assert VO.emit(fmt, K.KIND_14, r, cdev) is None
            out = np.full(1 << 17, 0xA5, np.uint8)
            need = C.c_size_t(12345)
            rc = fn(kx.ctx, fmt, K.KIND_14, r.ctypes.data, len(r), out.ctypes.data, len(out), C.byref(need))
            assert rc == B.E_UNSUPPORTED, k
            assert (out == 0xA5).all(), k  # nothing written
            rc = fn(kx.ctx, fmt, K.KIND_14, r.ctypes.data, len(r), None, 0, C.byref(need))  # the sizing call too
            assert rc == B.E_UNSUPPORTED, k
        out = np.full(1 << 17, 0xA5, np.uint8)
        rc = fn(kx.ctx, fmt, b"no-slash", good.ctypes.data, len(good), out.ctypes.data, len(out), C.byref(C.c_size_t()))
        assert rc == B.E_UNSUPPORTED and (out == 0xA5).all()
        assert fn(kx.ctx, 2, K.KIND_14, good.ctypes.data, len(good), None, 0, C.byref(C.c_size_t())) == B.E_INVALID
    # the key bytes past key_len and the reserved bytes are ignored
    noisy = good.copy()
    keys = np.frombuffer(noisy["key"].tobytes(), np.uint8).reshape(-1, 40).copy()
    for i in range(len(noisy)):
        keys[i, noisy["key_len"][i]:] = 0xEE
    noisy["key"] = keys.view("S40").reshape(-1)
    noisy["reserved"] = 0x7F
    assert kx.cdi_emit_vf_vgpu(K.FMT_YAML, noisy, K.KIND_14, cdev=cdev) == VO.emit(K.FMT_YAML, K.KIND_14, good, cdev)


@pytest.mark.parametrize("cdev", [False, True])
def test_sizing_nospace_and_timing(kx, cdev):
    recs = K.records(1000, seed=4)
    fn = _emit_raw(kx, cdev)
    doc = VO.emit(K.FMT_JSON, K.KIND_14, recs, cdev)
    need = C.c_size_t(0)
    rc = fn(kx.ctx, K.FMT_JSON, K.KIND_14, recs.ctypes.data, len(recs), None, 0, C.byref(need))
    assert (rc, need.value) == (B.E_NOSPACE, len(doc))
    out = np.zeros(len(doc) - 1, np.uint8)
    rc = fn(kx.ctx, K.FMT_JSON, K.KIND_14, recs.ctypes.data, len(recs), out.ctypes.data, len(out), C.byref(need))
    assert (rc, need.value) == (B.E_NOSPACE, len(doc))
    assert kx.cdi_emit_vf_vgpu(K.FMT_JSON, recs, K.KIND_14, cdev=cdev) == doc
    assert kx.timings()[B.T_EMIT] > 0
    back = recs if cdev else K.group_view(recs)
    rc, n, _ = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_14, 0, cdev=cdev, typed=True)  # out = NULL: the sizing call
    assert (rc, n) == (B.E_NOSPACE, 1000)
    rc, n, out = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_14, 999, cdev=cdev, typed=True)
    assert (rc, n) == (B.E_NOSPACE, 1000) and not out.tobytes().strip(b"\0")  # nothing written
    rc, n, out = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_14, 1000, cdev=cdev, typed=True)
    assert (rc, n) == (B.KXPU_OK, 1000) and out.tobytes() == back.tobytes()
    assert kx.timings()[B.T_EMIT] > 0
    assert len(doc) // B.CDI_FRAG_MIN >= 1000
    # a damaged document: a type ID with a leading zero, a key past 40 bytes, an unquoted value
    for old, new in ((b'"vgpu-type": "1",', b'"vgpu-type": "01",'), (b'"vgpu-type-key": "A"', b'"vgpu-type-key": "' + b"A" * 41 + b'"'),
                     (b'"vgpu-type": "1",', b'"vgpu-type": 1,'), (b'"vgpu-type": "1",', b'"vgpu-type": "0",')):
        assert old in doc
        rc, n, _ = kx.cdi_parse_raw(K.FMT_JSON, doc.replace(old, new, 1), K.KIND_14, 1000, cdev=cdev, typed=True)
        assert (rc, n) == (B.E_INVALID, -1), new
