"""CPU tests of the Prometheus metrics document (include/kxpu.h, kxpu_metrics_devices): the plain-Python writer against
hand-written documents (every family empty and not, every reason kind, each escape, UTF-8 repairs), against an
independent parser (prometheus_client) under hypothesis, the header's constants, and the host's document with no device."""
import ctypes as C

import pytest
from hypothesis import given, settings, strategies as st
from prometheus_client.parser import text_string_to_metric_families

import fake_sysfs
import pyref_metrics as PM
from kxpu_b200.binding import METRICS_HEADS, METRICS_REASONS

H1, H2, H3 = METRICS_HEADS[:3]
R = b"nvidia.com/GH100_H100_SXM5_80GB"


def doc(b):
    return PM.document(*b.arrays())


def test_header_constants():
    assert METRICS_REASONS == ("vfio-device-missing", "not-viable", "vfio-cdev-missing", "sriov", "reset", "pcie-aer",
                               "vgpu-type-changed")
    assert H1 == (b"# HELP kata_xpu_device_healthy Whether ListAndWatch reports the device Healthy (1) or Unhealthy (0).\n"
                  b"# TYPE kata_xpu_device_healthy gauge\n")
    assert H2 == (b"# HELP kata_xpu_device_unhealthy_reason Why the plugin reports the device Unhealthy, one sample per "
                  b"reason.\n# TYPE kata_xpu_device_unhealthy_reason gauge\n")
    assert H3 == (b"# HELP kata_xpu_pcie_aer_errors The highest TOTAL_ERR count the device's aer_dev files reported at the "
                  b"last read.\n# TYPE kata_xpu_pcie_aer_errors gauge\n")
    assert METRICS_HEADS[3].endswith(b"# TYPE kata_xpu_sysfs_reads_total counter\n")
    assert METRICS_HEADS[4].endswith(b"# TYPE kata_xpu_allocate_validations_total counter\n")


def test_no_device_is_empty():
    assert doc(PM.Builder()) == b""


def test_healthy_only():
    b = PM.Builder().add(R, 41, b"0000:41:00.0").add(R, 7, b"0000:07:00.0", healthy=0)
    assert doc(b) == H1 + (b'kata_xpu_device_healthy{resource="nvidia.com/GH100_H100_SXM5_80GB",device="41",'
                           b'address="0000:41:00.0"} 1\n'
                           b'kata_xpu_device_healthy{resource="nvidia.com/GH100_H100_SXM5_80GB",device="7",'
                           b'address="0000:07:00.0"} 0\n')


def test_every_kind_in_order():
    why = [(k, b"why %d" % k) for k in range(7)]
    why[0] = (0, b"")
    b = PM.Builder().add(b"r/x", 3, b"a", healthy=0, reasons=why)
    want = H1 + b'kata_xpu_device_healthy{resource="r/x",device="3",address="a"} 0\n' + H2
    for k, d in why:
        want += (b'kata_xpu_device_unhealthy_reason{resource="r/x",device="3",address="a",reason="%s",detail="%s"} 1\n'
                 % (METRICS_REASONS[k].encode(), d))
    assert doc(b) == want


def test_aer_family():
    b = PM.Builder().add(b"r/x", 3, b"a", aer_fatal=0).add(b"r/x", 4, b"b").add(b"r/x", 5, b"c", aer_fatal=7,
                                                                                   aer_nonfatal=2 ** 64 - 2)
    want = (H1 + b'kata_xpu_device_healthy{resource="r/x",device="3",address="a"} 1\n'
            b'kata_xpu_device_healthy{resource="r/x",device="4",address="b"} 1\n'
            b'kata_xpu_device_healthy{resource="r/x",device="5",address="c"} 1\n' + H3 +
            b'kata_xpu_pcie_aer_errors{resource="r/x",device="3",address="a",severity="fatal"} 0\n'
            b'kata_xpu_pcie_aer_errors{resource="r/x",device="5",address="c",severity="fatal"} 7\n'
            b'kata_xpu_pcie_aer_errors{resource="r/x",device="5",address="c",severity="nonfatal"} 18446744073709551614\n')
    assert doc(b) == want
    only_nonfatal = PM.Builder().add(b"r/x", 3, b"a", aer_nonfatal=1)
    assert doc(only_nonfatal).endswith(H3 + b'kata_xpu_pcie_aer_errors{resource="r/x",device="3",address="a",'
                                             b'severity="nonfatal"} 1\n')


@pytest.mark.parametrize("raw,want", [
    (b'a"b', b'a\\"b'),
    (b"a\\b", b"a\\\\b"),
    (b"a\nb", b"a\\nb"),
    (b"\r\t", b"\r\t"),                                       # only three bytes are escaped
    (b"", b""),
    (b"\xc3\xa9", b"\xc3\xa9"),                               # 2-byte sequence kept
    (b"\xe2\x82\xac", b"\xe2\x82\xac"),                       # 3-byte
    (b"\xf0\x9f\x98\x80", b"\xf0\x9f\x98\x80"),               # 4-byte
    (b"\xf0\x9f\x98", b"\xef\xbf\xbd"),                       # truncated 4-byte: one maximal subpart
    (b"\xe2\x82", b"\xef\xbf\xbd"),                           # truncated 3-byte
    (b"\xe2\x82x", b"\xef\xbf\xbdx"),
    (b"\xc0\xaf", b"\xef\xbf\xbd" * 2),                       # overlong: C0 is no lead
    (b"\xe0\x80\xaf", b"\xef\xbf\xbd" * 3),                   # overlong 3-byte
    (b"\xf0\x8f\xbf\xbf", b"\xef\xbf\xbd" * 4),               # overlong 4-byte
    (b"\xed\xa0\x80", b"\xef\xbf\xbd" * 3),                   # surrogate U+D800
    (b"\xed\x9f\xbf", b"\xed\x9f\xbf"),                       # U+D7FF is fine
    (b"\xf4\x90\x80\x80", b"\xef\xbf\xbd" * 4),               # above U+10FFFF
    (b"\xf5\x80", b"\xef\xbf\xbd" * 2),
    (b"\x80\x80\x80\x80\x80", b"\xef\xbf\xbd" * 5),           # lone continuation bytes
    (b"\xff\"", b'\xef\xbf\xbd\\"'),
])
def test_label_escapes_and_repairs(raw, want):
    assert PM.label(raw) == want
    b = PM.Builder().add(b"r/x", 1, b"a", healthy=0, reasons=[(1, raw)])
    assert doc(b).endswith(b'reason="not-viable",detail="%s"} 1\n' % want)


def _parsed(text):
    return [(s.name, dict(s.labels), s.value) for f in text_string_to_metric_families(text) for s in f.samples]


_bytes = st.binary(max_size=48) | st.lists(st.sampled_from([b"a", b"\\", b'"', b"\n", b"\xc3\xa9", b"\xe2\x82",
                                                            b"\xf0\x9f\x98\x80", b"\xed\xa0\x80", b"\x80", b"\xff"]),
                                           max_size=12).map(b"".join)


@settings(max_examples=300, deadline=None)
@given(st.lists(st.tuples(_bytes, st.integers(0, 2 ** 32 - 1), _bytes, st.integers(0, 1),
                          st.lists(st.tuples(st.integers(0, 6), _bytes), max_size=4),
                          st.sampled_from([None, 0, 1, 2 ** 64 - 2]), st.sampled_from([None, 0, 5])), max_size=6))
def test_parser_reads_back_every_sample(devices):
    b, want = PM.Builder(), []
    for res, grp, addr, ok, why, fat, nonfat in devices:
        kinds = sorted({k: d for k, d in why}.items())
        b.add(res, grp, addr, ok, kinds, PM.METRICS_NO_VALUE if fat is None else fat,
              PM.METRICS_NO_VALUE if nonfat is None else nonfat)
        lab = dict(resource=res.decode("utf-8", "replace"), device=str(grp), address=addr.decode("utf-8", "replace"))
        want.append((0, "kata_xpu_device_healthy", lab, ok))
        for k, d in kinds:
            want.append((1, "kata_xpu_device_unhealthy_reason",
                         dict(lab, reason=METRICS_REASONS[k], detail=d.decode("utf-8", "replace")), 1))
        for sev, v in (("fatal", fat), ("nonfatal", nonfat)):
            if v is not None:
                want.append((2, "kata_xpu_pcie_aer_errors", dict(lab, severity=sev), v))
    text = doc(b)
    assert text == b"" or text.endswith(b"\n")
    got = _parsed(text.decode("utf-8"))
    want = [w[1:] for w in sorted(want, key=lambda w: w[0])]  # family-major, device order within (a stable sort)
    assert [(n, l) for n, l, _ in got] == [(n, l) for n, l, _ in want]
    assert [float(v) for _, _, v in got] == [float(v) for _, _, v in want]


@pytest.fixture
def hp(tmp_path):
    base = fake_sysfs.make_tree(str(tmp_path), [dict(bdf="0000:03:00.0", group=30, vendor=b"0x10de\n",
                                                     device=b"0x2330\n", driver="vfio-pci")])
    p = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), base, str(tmp_path / "pci.ids"), str(tmp_path) + "/")
    try:
        yield p
    finally:
        p.close()


def host_metrics(hp):
    hp.L.kxh_metrics.restype = C.c_int
    hp.L.kxh_metrics.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t]
    buf, n, err = C.create_string_buffer(1 << 22), C.c_size_t(0), C.create_string_buffer(512)
    rc = hp.L.kxh_metrics(hp.h, buf, len(buf), C.byref(n), err, len(err))
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return buf.raw[:n.value]


def test_host_without_plugins_has_only_its_counters(hp):
    # no walk yet: no plugin, no device, so no family of the GPU's; the counters are all there, at zero
    assert host_metrics(hp) == PM.counters()
    assert host_metrics(hp) == PM.counters()  # and a scrape changes nothing


def test_long_reason_is_cut():
    """a reason over KXPU_METRICS_STRING_MAX bytes is cut on the host at a UTF-8 sequence boundary"""
    L = fake_sysfs.host_lib()
    L.kxh_metrics_cut.restype = C.c_size_t
    L.kxh_metrics_cut.argtypes = [C.c_char_p, C.c_size_t]
    assert L.kxh_metrics_cut(b"x" * 4096, 4096) == 4096
    assert L.kxh_metrics_cut(b"x" * 5000, 5000) == 4096
    assert L.kxh_metrics_cut(b"x" * 4095 + b"\xe2\x82\xac", 4098) == 4095  # the euro sign would be split
    assert L.kxh_metrics_cut(b"x" * 4094 + b"\xe2\x82\xac", 4097) == 4094
    assert L.kxh_metrics_cut(b"x" * 4093 + b"\xe2\x82\xac", 4096) == 4096
    assert L.kxh_metrics_cut(b"\x80" * 5000, 5000) == 4096  # no lead in reach: cut at the limit
