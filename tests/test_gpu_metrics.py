"""GPU tests of kxpu_metrics_devices against the plain-Python writer (tests/pyref_metrics.py): byte for byte from 0 to
2^20 devices, details at the lengths and offsets where the warp's 32-byte steps turn, every escape and UTF-8 repair at
every offset modulo 32, the sizing call one byte short, and every refusal with the output left untouched."""
import numpy as np
import pytest

import pyref_metrics as PM
from kxpu_b200.binding import E_NOSPACE, KXPU_OK, METRICS_NO_VALUE, KxpuError

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -7
R = b"nvidia.com/GH100_H100_SXM5_80GB"


def check(kx, b):
    devs, strings, reasons = b.arrays()
    assert kx.metrics_devices(devs, strings, reasons) == PM.document(devs, strings, reasons)


def test_empty(kx):
    check(kx, PM.Builder())


@pytest.mark.parametrize("n", [1, 7, 8, 9, 4095, 4096, 4097, 65537])
def test_sizes(kx, n):
    b = PM.Builder()
    for i in range(n):
        why = [(k, b"0000:%02x:00.0 reason %d" % (i & 0xff, k)) for k in range(7) if (i >> k) & 1 and i % 3 == 0]
        b.add(R, i * 7919 % 1000003, b"0000:%02x:00.0" % (i & 0xff), int(not why), why,
              i if i % 5 == 0 else METRICS_NO_VALUE, 2 ** 64 - 2 - i if i % 7 == 0 else METRICS_NO_VALUE)
    check(kx, b)


@pytest.mark.parametrize("length", [0, 1, 31, 32, 33, 63, 64, 65, 4095, 4096])
def test_detail_lengths(kx, length):
    rng = np.random.default_rng(length)
    b = PM.Builder()
    b.add(R, 1, b"a", 0, [(1, bytes(rng.integers(0x20, 0x7f, length, np.uint8)))])
    b.add(R, 2, b"b", 0, [(3, b"\xff" * length), (6, b'"\\\n' * (length // 3) + b"x" * (length % 3))])
    b.add(R, 3, b"c" * length, 1, [], 5, 6)
    check(kx, b)


SEQS = [b'"', b"\\", b"\n", b"\xc3\xa9", b"\xe2\x82\xac", b"\xf0\x9f\x98\x80", b"\xf0\x9f\x98", b"\xe2\x82", b"\xc3",
        b"\x80", b"\xff", b"\xc0\xaf", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"\xe0\x80\xaf"]


@pytest.mark.parametrize("seq", SEQS)
def test_every_offset(kx, seq):
    """the sequence at every offset 0..95 of a detail, of the resource and of the address, so it meets the 32-byte steps
    of the warp at every phase and straddles their edges"""
    b = PM.Builder()
    for off in range(96):
        d = b"x" * off + seq + b"y" * (70 - off % 40)
        b.add(b"r/" + b"q" * off + seq, off, b"z" * (off % 40) + seq, 0, [(0, b""), (2, d), (5, seq * (off % 5))], off)
    check(kx, b)


def test_random_bytes(kx):
    rng = np.random.default_rng(7)
    b = PM.Builder()
    for i in range(2000):
        why = [(k, bytes(rng.integers(0, 256, int(rng.integers(0, 200)), np.uint8))) for k in range(7) if rng.random() < 0.2]
        b.add(bytes(rng.integers(0, 256, int(rng.integers(0, 40)), np.uint8)), int(rng.integers(0, 2 ** 32)),
              bytes(rng.integers(0x80, 256, int(rng.integers(0, 40)), np.uint8)), int(not why), why)
    check(kx, b)


def test_2_20_devices(kx):
    from kxpu_b200.workloads import metrics_devices
    devs, strings, reasons = metrics_devices(1 << 20)
    assert kx.metrics_devices(devs, strings, reasons) == PM.document(devs, strings, reasons)


def test_cap_one_short(kx):
    b = PM.Builder().add(R, 41, b"0000:41:00.0", 0, [(1, b"why \xff")], 3)
    devs, strings, reasons = b.arrays()
    want = PM.document(devs, strings, reasons)
    rc, need = kx.metrics_devices_raw(devs, strings, reasons, None, 0)
    assert rc == E_NOSPACE and need == len(want)
    out = np.full(need + 8, 0xA5, np.uint8)
    rc, got = kx.metrics_devices_raw(devs, strings, reasons, out, need - 1)
    assert rc == E_NOSPACE and got == need and (out == 0xA5).all()
    rc, got = kx.metrics_devices_raw(devs, strings, reasons, out, need)
    assert rc == KXPU_OK and got == need and out[:need].tobytes() == want and (out[need:] == 0xA5).all()


def _refusal(kx, devs, strings, reasons, status):
    out = np.full(1 << 16, 0xA5, np.uint8)
    rc, _ = kx.metrics_devices_raw(devs, strings, reasons, out, out.size)
    assert rc == status
    assert (out == 0xA5).all()


def _base():
    return PM.Builder().add(R, 1, b"a", 0, [(1, b"x"), (4, b"y")]).add(R, 2, b"b", 1).arrays()


@pytest.mark.parametrize("case", ["resource", "address", "detail", "healthy", "run", "run_off", "kind", "repeat", "order"])
def test_invalid(kx, case):
    devs, strings, reasons = _base()
    big = len(strings) + 1
    if case == "resource":
        devs[1]["resource_off"] = len(strings) - 1; devs[1]["resource_len"] = 2
    elif case == "address":
        devs[0]["address_off"] = 2 ** 64 - 1; devs[0]["address_len"] = 2
    elif case == "detail":
        reasons[1]["detail_off"] = big
    elif case == "healthy":
        devs[1]["healthy"] = 2
    elif case == "run":
        devs[1]["reason_off"] = 1; devs[1]["reason_count"] = 2
    elif case == "run_off":
        devs[1]["reason_off"] = 2 ** 64 - 1; devs[1]["reason_count"] = 1
    elif case == "kind":
        reasons[1]["kind"] = 7
    elif case == "repeat":
        reasons[1]["kind"] = 1
    elif case == "order":
        reasons[0]["kind"], reasons[1]["kind"] = 4, 1
    _refusal(kx, devs, strings, reasons, E_INVALID)


@pytest.mark.parametrize("case", ["detail", "resource", "address"])
def test_unsupported_strings(kx, case):
    long = b"x" * 4097
    b = PM.Builder()
    if case == "detail":
        b.add(R, 1, b"a", 0, [(1, long)])
    elif case == "resource":
        b.add(long, 1, b"a")
    else:
        b.add(R, 1, long)
    _refusal(kx, *b.arrays(), E_UNSUPPORTED)
    ok = PM.Builder().add(R, 1, b"a" * 4096, 0, [(1, b"x" * 4096)])
    check(kx, ok)


def test_unsupported_sizes(kx):
    import ctypes as C
    n = C.c_size_t(0)
    out = np.full(64, 0xA5, np.uint8)
    dev = np.zeros(1, PM.METRICDEV_DTYPE)
    assert kx.L.kxpu_metrics_devices(kx.ctx, dev.ctypes.data, 1 << 28, None, 0, None, 0, out.ctypes.data, 64, C.byref(n)) == E_UNSUPPORTED
    assert (out == 0xA5).all()
    # 2^40 bytes and more: every device names the same 4096-byte strings, 2^22 devices with seven reasons each
    devs = np.zeros(1 << 22, PM.METRICDEV_DTYPE)
    devs["resource_len"] = devs["address_len"] = 4096
    devs["reason_count"] = 7
    devs["aer_fatal"] = devs["aer_nonfatal"] = METRICS_NO_VALUE
    reasons = np.zeros(7, PM.METRICREASON_DTYPE)
    reasons["kind"] = np.arange(7)
    reasons["detail_len"] = 4096
    strings = b"\xff" * 4096
    _refusal(kx, devs, strings, reasons, E_UNSUPPORTED)


def test_errors_raise(kx):
    devs, strings, reasons = _base()
    reasons[0]["kind"] = 9
    with pytest.raises(KxpuError):
        kx.metrics_devices(devs, strings, reasons)


def test_null_arguments(kx):
    """KXPU_E_INVALID for every NULL the header names, with nothing written"""
    import ctypes as C
    devs, strings, reasons = _base()
    sb = np.frombuffer(strings, np.uint8)
    out = np.full(1 << 12, 0xA5, np.uint8)
    n = C.c_size_t(7)
    f = kx.L.kxpu_metrics_devices
    args = [kx.ctx, devs.ctypes.data, len(devs), sb.ctypes.data, len(sb), reasons.ctypes.data, len(reasons),
            out.ctypes.data, out.size, C.byref(n)]
    for k in (0, 1, 3, 5, 9):  # ctx, devs, strings, reasons, len
        a = list(args)
        a[k] = None
        assert f(*a) == E_INVALID
        assert (out == 0xA5).all() and n.value == 7
    assert f(*args) == KXPU_OK and n.value == len(PM.document(devs, strings, reasons))
