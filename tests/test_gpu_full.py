"""SURVEY 8(f) row 4: subsystem rows and the class / subclass / prog-if section, GPU vs oracle (kxo_full_build)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def check_full(kx, oracle, text):
    buf = np.frombuffer(text, np.uint8)
    d = kx.dev_alloc(max(len(buf), 16))
    if len(buf):
        kx.upload(d, buf)
    tab = kx.pciids_load_device(d, len(buf))
    full = kx.full_load_device(d, len(buf), tab)
    try:
        for kind in (0, 1, 2):
            want = oracle.full_build(text, kind)
            keys, offs = kx.full_export(full, kind)
            assert np.array_equal(keys, want["key"]) and np.array_equal(offs, want["line_off"]), kind
            if len(want):
                pick = want[:: max(1, len(want) // 400)]
                q = np.concatenate([pick["key"], pick["key"] ^ np.uint64(1 << 5), np.array([0, 1 << 63, (1 << 64) - 2], np.uint64)])
                got = kx.full_lookup(full, kind, q)
                table = dict(zip(want["key"].tolist(), want["line_off"].tolist()))
                exp = np.array([table.get(int(k), -1) for k in q], np.int64)
                assert np.array_equal(got, exp), kind
    finally:
        kx.full_free(full)
        tab.free()
        kx.dev_free(d)


def test_real_pci_ids_full_model(kx, oracle, pci_text):
    want = [len(oracle.full_build(pci_text, k)) for k in (0, 1, 2)]
    assert want == [2388, 16297, 210]  # SURVEY.md 8(a) A0: vendors, subsystem lines, 22 + 114 + 74 class-section lines
    check_full(kx, oracle, pci_text)


def test_full_model_first_occurrence_and_edges(kx, oracle, pci_text, workloads):
    cut = pci_text.find(b"\n", 1400000) + 1
    check_full(kx, oracle, pci_text * 2)                         # every block twice: the first copy wins at every level
    check_full(kx, oracle, pci_text[700000:cut] + pci_text)      # later vendors first, class section twice
    texts = [b"", b"\n", b"\t\t1234 5678  orphan\n", b"1234  V\n\t0001  d\n\t\t1111 2222  s\n\t\t1111 2222  dup\n\t0001  dupdev\n\t\t3333 4444  lost\n",
             b"C 01  cls\n\t02  sub\n\t\t03  pi\n\t\t03  dup\n\t02  dupsub\n\t\t04  lost\nC 01  again\n\t05  lost\n",
             b"1234  V\n\t0001  d\n#c\n\t\t1111 2222  after comment\n\n\t\t5555 6666  after blank\n",
             b"1234  V\r\n\t0001  d\r\n\t\t1111 2222  crlf\r\n", b"C 0g  bad\n\t01  x\n1234  V\n\t00  short\n\t\t1111 2222  under short\n",
             b"1234  V\n\t0001  d\n\t\t1111  one id only\n\t\t11112222  no blank\n\t\t1111 222  short\n\t\t1111 2222\n"]
    for t in texts:
        check_full(kx, oracle, t)
    # lines whose governing lines sit one or many 2 KiB chunks back
    big = b"abcd  Vendor\n\t0001  dev\n" + b"".join(b"\t\t%04x %04x  subsystem number %d\n" % (i >> 8, i & 0xffff, i) for i in range(9000))
    big += b"C ff  class\n\t01  sub\n" + b"".join(b"\t\t%02x  prog-if %d\n" % (i & 0xff, i) for i in range(400))
    check_full(kx, oracle, big)
    # more subsystem rows than the first subsystem hash table (2^17 slots) and more prog-if rows than the first
    # prog-if table (2^12 slots) hold: both are grown x4 and built again
    text = workloads.synthetic_pci_ids(512, 64, subs_per_dev=8).tobytes()
    classes = b"".join(b"C %02x  Class %d\n\t%02x  Subclass\n" % (c, c, c) + b"".join(b"\t\t%02x  Prog-if %d\n" % (p, p) for p in range(256))
                       for c in range(20))
    text += classes
    assert len(oracle.full_build(text, 1)) == 262144 > (1 << 17)
    progifs = oracle.full_build(text, 2)
    assert int(((progifs["key"] >> np.uint64(24)) == 3).sum()) == 5120 > (1 << 12)
    check_full(kx, oracle, text)


def test_full_model_fuzz(kx, oracle):
    rng = np.random.default_rng(12)
    pool = [b"%04x  V\n", b"\t%04x  D\n", b"\t\t%04x %04x  S\n", b"C %02x  K\n", b"\t%02x  SC\n", b"\t\t%02x  PI\n", b"# c\n", b"\n", b"zz\n", b"\t\n",
            b"\t\t\n"]
    for trial in range(40):
        parts = []
        for _ in range(int(rng.integers(1, 2500))):
            f = pool[int(rng.integers(0, len(pool)))]
            k = f.count(b"%")
            parts.append(f % tuple(int(rng.integers(0, 6)) for _ in range(k)) if k else f)
        check_full(kx, oracle, b"".join(parts))
