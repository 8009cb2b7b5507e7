"""CPU tests: the oracle against its pins (golden.json), the format goldens of SURVEY.md
8a-fmt and independent Python restatements (pyref.py, pyref_full.py)."""
import hashlib
import json
import os

import numpy as np
import pytest
import yaml
from hypothesis import given, settings, strategies as st

import full_texts
import pyref
import pyref_full
from conftest import GOLDEN
from pyref import MAX_TOKEN


def test_pci_ids_fixture_pinned(pci_text, golden):
    assert len(pci_text) == golden["pci_ids_bytes"] == 1458186
    assert hashlib.sha256(pci_text).hexdigest() == golden["pci_ids_sha256"]


def test_table_dump_matches_self_pins(oracle, pci_text, oracle_rows, golden):
    assert len(oracle_rows) == golden["rows"] == 18856
    dump = b"".join(b"%04x:%04x\t%s\n" % (r["key"] >> 16, r["key"] & 0xFFFF, oracle.row_name(pci_text, int(r["line_off"])))
                    for r in oracle_rows)
    assert len(dump) == golden["dump_bytes"]
    assert hashlib.sha256(dump).hexdigest() == golden["dump_sha256"]
    nv = b"".join(l + b"\n" for l in dump.split(b"\n") if l.startswith(b"10de:"))
    assert nv.count(b"\n") == golden["nvidia_rows"] == 1859
    assert hashlib.sha256(nv).hexdigest() == golden["nvidia_dump_sha256"]


def test_spot_values(oracle, pci_text, golden):
    for k, want in golden["spots"].items():
        off, nm = oracle.device_name(pci_text, int(k, 16))
        assert off == want["line_off"]
        assert (None if nm is None else nm.decode()) == want["name"]
    # SURVEY.md 8(a) A7 examples
    assert oracle.device_name(pci_text, 0x10de2330)[1] == b"GH100_H100_SXM5_80GB"
    assert oracle.device_name(pci_text, 0x10de28e0)[1] == b"AD107M_GEFORCE_RTX_4060_MAXQ___MOBILE"
    assert oracle.device_name(pci_text, 0x10de2901) == (-1, None)


def test_names_bulk_equals_row_name(oracle, pci_text, oracle_rows):
    """names_bulk (one call for all rows, the checker of the large-table GPU tests) == row_name for every
    row of the real file, and == the Python sanitiser on a sample; edge lines too."""
    offs_in = oracle_rows["line_off"]
    blob, offs = oracle.names_bulk(pci_text, offs_in)
    assert len(offs) == len(offs_in) + 1 and offs[0] == 0 and offs[-1] == len(blob)
    for i, o in enumerate(offs_in.tolist()):
        assert blob[offs[i]:offs[i + 1]] == oracle.row_name(pci_text, o), i
    rng = np.random.default_rng(5)
    for i in rng.choice(len(offs_in), 300, replace=False).tolist():
        o = int(offs_in[i])
        line = pci_text[o:pci_text.index(b"\n", o)].removesuffix(b"\r")
        assert blob[offs[i]:offs[i + 1]] == pyref.sanitise(line[5:])
    # short, empty, CRLF and unterminated lines; the same line twice; no lines at all
    text = b"10de  V\n\t0001\n\t0002  a b\r\n\t00\n\t0003  \xc4\xb1x/y"
    lo = np.array([8, 14, 26, 8, 30, 14], np.uint64)
    blob, offs = oracle.names_bulk(text, lo)
    assert [blob[offs[i]:offs[i + 1]] for i in range(len(lo))] == [oracle.row_name(text, int(o)) for o in lo]
    assert [blob[offs[i]:offs[i + 1]] for i in range(len(lo))] == [b"", b"A_B", b"", b"", b"IX_Y", b"A_B"]
    blob, offs = oracle.names_bulk(text, np.empty(0, np.uint64))
    assert blob == b"" and offs.tolist() == [0]


def test_literal_scan_equals_single_pass_table(oracle, pci_text, oracle_rows):
    """Every key of the one-pass table resolves, by the literal getDeviceName scan, to the
    same line; sampled (the literal scan is O(file) per key)."""
    rng = np.random.default_rng(7)
    idx = rng.choice(len(oracle_rows), 400, replace=False)
    for i in idx:
        off, _ = oracle.device_name(pci_text, int(oracle_rows["key"][i]))
        assert off == int(oracle_rows["line_off"][i])


def test_literal_scan_vs_python_restatement(oracle, pci_text, oracle_rows):
    rng = np.random.default_rng(11)
    keys = [int(k) for k in oracle_rows["key"][rng.choice(len(oracle_rows), 40, replace=False)]]
    keys += [0x10de2901, 0xffff0000, 0x80860000, 0x0001ffff, 0x00010000]
    for k in keys:
        v, d = b"%04x" % (k >> 16), b"%04x" % (k & 0xFFFF)
        assert oracle.device_name(pci_text, k) == pyref.get_device_name(pci_text, v, d)


EDGE_TEXTS = [
    b"",
    b"\n",
    b"10de  NVIDIA\n\t2330  GH100 [H100 SXM5 80GB]\n",
    b"10de  NVIDIA\n\t2330  GH100 [H100 SXM5 80GB]",            # no trailing newline
    b"10de  NVIDIA\r\n\t2330  A.b/c  d\r\n",                     # CRLF
    b"10de  NV\n# c\n\t0001  one\n\n\t0002  unreachable\n",      # blank line ends the block
    b"10de  first\n\t0001  a\n10df  x\n10de  again\n\t0002  hidden\n",  # only the first anchor counts
    b"\t0001  orphan\n10de  NV\n\t0001  real\n\t0001  dup\n",
    b"10de\n\t0001\n",                                           # empty names
    b"10deXYZ\n\t00012  id-prefix match\n",                      # raw prefix semantics
    b"# only comments\n#\n",
    b"C 03  Display\n\t00  VGA\n\t\t00  x\n",
]


@pytest.mark.parametrize("text", EDGE_TEXTS)
def test_edge_texts(oracle, text):
    rows = oracle.table_build(text)
    for k in [0x10de2330, 0x10de0001, 0x10de0002, 0x10df0001, 0x10de0001, 0x00000000]:
        v, d = b"%04x" % (k >> 16), b"%04x" % (k & 0xFFFF)
        got = oracle.device_name(text, k)
        assert got == pyref.get_device_name(text, v, d), (text, hex(k))
        hit = rows[rows["key"] == k]
        assert (len(hit) == 1 and int(hit["line_off"][0]) == got[0]) or (len(hit) == 0 and got[0] == -1)


def test_too_long_line_stops_scan(oracle):
    long_line = b"#" + b"x" * 65535  # 65536 content bytes -> bufio.ErrTooLong
    ok_line = b"#" + b"x" * 65534
    t1 = b"10de  NV\n\t0001  a\n" + ok_line + b"\n\t0002  b\n"
    t2 = b"10de  NV\n\t0001  a\n" + long_line + b"\n\t0002  b\n"
    assert oracle.device_name(t1, 0x10de0002)[1] == b"B"
    assert oracle.device_name(t2, 0x10de0001)[1] == b"A"
    assert oracle.device_name(t2, 0x10de0002) == (-1, None)
    for t in (t1, t2):
        for k in (0x10de0001, 0x10de0002):
            assert oracle.device_name(t, k) == pyref.get_device_name(t, b"%04x" % (k >> 16), b"%04x" % (k & 0xFFFF))


SANITISE_CASES = [
    (b"  GH100 [H100 SXM5 80GB]", b"GH100_H100_SXM5_80GB"),
    (b"  AD107M [GeForce RTX 4060 Max-Q / Mobile]", b"AD107M_GEFORCE_RTX_4060_MAXQ___MOBILE"),
    (b"  Integrated Lights Out  Processor", b"INTEGRATED_LIGHTS_OUT_PROCESSOR"),
    (b"  88W8997 2.4/5 GHz Dual-Band 2x2 Wi-Fi\xc2\xae 5 (802.11ac) + Bluetooth\xc2\xae 5.3 Solution",
     b"88W8997_2_4_5_GHZ_DUALBAND_2X2_WIFI_5_802_11AC__BLUETOOTH_5_3_SOLUTION"),
    (b"", b""), (b"   ", b""), (b" a\tb \x0b c ", b"A_B__C"),
    (b"x \xc2\xa0", b"X"),                 # trailing NBSP is Unicode space: trimmed with the blank before it
    (b"\xc2\xa0 x", b"X"),
    (b"a\xc2\xa0b", b"AB"),                # interior NBSP is not RE2 \s: deleted
    (b"d\xc4\xb1g \xc5\xbf", b"DIG_S"),    # U+0131 -> I, U+017F -> S
    (b"\xff\xfe ok", b"_OK"),              # invalid UTF-8 is not space: kept by TrimSpace, deleted at the end
    (b"stra\xc3\x9fe", b"STRAE"),          # sharp s has no simple upper-case: deleted
    (b"a__b..c//d", b"A__B__C__D"),
    (b"\xe2\x80\x83em space\xe3\x80\x80", b"EM_SPACE"),
]


@pytest.mark.parametrize("rest,want", SANITISE_CASES)
def test_sanitise_cases(oracle, rest, want):
    assert oracle.sanitise(rest) == want
    assert pyref.sanitise(rest) == want


@settings(max_examples=300, deadline=None)
@given(st.text(alphabet=st.sampled_from(list(" \t\r\x0b\x0cabzAZ09_./-[]() ıſßé ®")), max_size=24))
def test_sanitise_property(oracle, s):
    b = s.encode()
    if b"\n" in b:
        return
    assert oracle.sanitise(b) == pyref.sanitise(b)


def full_rows_equal(oracle, text):
    for kind in (0, 1, 2):
        want = oracle.full_build(text, kind)
        assert list(zip(want["key"].tolist(), want["line_off"].tolist())) == pyref_full.full_build(text, kind), kind


def test_full_model_real_file_vs_python(oracle, pci_text):
    """kxo_full_build == pyref_full on the real file: every vendor, subsystem and class-section row."""
    assert [len(pyref_full.full_build(pci_text, k)) for k in (0, 1, 2)] == [2388, 16297, 210]
    full_rows_equal(oracle, pci_text)
    full_rows_equal(oracle, pci_text[700000:pci_text.find(b"\n", 1400000) + 1] + pci_text)


def test_full_model_edge_texts_vs_python(oracle):
    texts = full_texts.EDGE_TEXTS + [full_texts.ALL_ONES, full_texts.all_ones_first(), full_texts.seam_text()]
    texts += full_texts.lookback_texts() + full_texts.length_texts()
    for t in texts:
        full_rows_equal(oracle, t)
    want = oracle.full_build(full_texts.ALL_ONES, 1)
    assert want["key"].tolist() == full_texts.ALL_ONES_KEYS and want["line_off"].tolist() == full_texts.ALL_ONES_OFFS


def test_full_model_cutoff_vs_python(oracle):
    """A line of 64 KiB or more (a trailing '\\r' counts) ends the scan: no row of any kind at or behind it."""
    for text, uncut, kept in full_texts.cutoff_texts():
        full_rows_equal(oracle, text)
        full_rows_equal(oracle, uncut)
        at = text.index(b"x" * 1000) - 1
        got = [oracle.full_build(text, k) for k in (0, 1, 2)]
        allr = [oracle.full_build(uncut, k) for k in (0, 1, 2)]
        if kept:
            assert [len(g) for g in got] == [len(a) for a in allr]
        else:
            assert all((g["line_off"] < at).all() for g in got)
            assert sum(len(g) for g in got) < sum(len(a) for a in allr)


FULL_IDS = [b"0000", b"0001", b"00ff", b"abcd", b"fffe", b"ffff", b"00FF", b"ABCD", b"FFFE", b"FFFF"]
FULL_IDS2 = [b"00", b"01", b"ff", b"FF", b"0g", b"a"]


@st.composite
def full_model_text(draw):
    """blocks of a top-level line and the lines that follow it, drawn from every line kind of both sections, their
    malformed forms (uppercase, invalid or too few digits, three tabs), comments, blank lines and CRLF endings"""
    i4, i2 = st.sampled_from(FULL_IDS), st.sampled_from(FULL_IDS2)
    top = st.one_of(
        st.tuples(i4).map(lambda t: t[0] + b"  V"),
        st.tuples(i2).map(lambda t: b"C " + t[0] + b"  K"),
        st.tuples(i2, st.sampled_from([b"c ", b"C\t", b"C  ", b"C"])).map(lambda t: t[1] + t[0]),
        st.sampled_from([b"C ", b"C 0", b"ffff", b"fff", b"", b"zz"]),
    )
    body = st.one_of(
        st.tuples(i4).map(lambda t: b"\t" + t[0] + b"  D"),
        st.tuples(i4, i4).map(lambda t: b"\t\t" + t[0] + b" " + t[1] + b"  S"),
        st.tuples(i4, i4).map(lambda t: b"\t\t" + t[0] + b" " + t[1]),
        st.tuples(i2).map(lambda t: b"\t" + t[0] + b"  SC"),
        st.tuples(i2).map(lambda t: b"\t\t" + t[0] + b"  PI"),
        st.tuples(i4, st.integers(0, 3)).map(lambda t: b"\t" + t[0][:t[1]]),
        st.tuples(i4, i4, st.integers(0, 3)).map(lambda t: b"\t\t" + t[0] + b" " + t[1][:t[2]]),
        st.tuples(i4, st.integers(0, 3)).map(lambda t: b"\t\t" + t[0][:t[1]]),
        st.tuples(i4, i4, st.sampled_from([b"", b"\t", b"x"])).map(lambda t: b"\t\t" + t[0] + t[2] + t[1]),
        st.tuples(i4, i4, st.sampled_from([b"\t\t\t", b"\t\t\t\t"])).map(lambda t: t[2] + t[0] + b" " + t[1]),
        st.sampled_from([b"\t", b"\t\t", b"# c", b"#", b"#\tffff ffff"]),
    )
    blocks = draw(st.lists(st.tuples(top, st.lists(body, max_size=12)), max_size=10))
    endings = st.sampled_from([b"\n", b"\n", b"\r\n"])
    lines = [(l, draw(endings)) for t, b in blocks for l in [t] + b]
    if lines and draw(st.integers(0, 7)) == 0:  # now and then one line of 64 KiB - 1 (kept) or 64 KiB (the scan stops)
        long = draw(st.sampled_from([b"#" + b"x" * (MAX_TOKEN - 2), b"#" + b"x" * (MAX_TOKEN - 1), b"ffff" + b"x" * (MAX_TOKEN - 4)]))
        lines.insert(draw(st.integers(0, len(lines))), (long, draw(st.sampled_from([b"\n", b"\r\n"]))))
    text = b"".join(l + e for l, e in lines)
    return text[:-1] if draw(st.booleans()) and text else text


@settings(max_examples=400, deadline=None)
@given(full_model_text())
def test_full_model_property_vs_python(oracle, text):
    full_rows_equal(oracle, text)


def test_cdi_goldens_cfg1(oracle, workloads):
    devs = np.zeros(1, dtype=oracle.CDIDEV_DTYPE)
    devs["bdf"], devs["iommu_group"], devs["index"] = b"0000:c1:00.0", 214, 0
    y = oracle.cdi_emit(0, devs)
    j = oracle.cdi_emit(1, devs)
    assert y == open(os.path.join(GOLDEN, "cfg1.yaml"), "rb").read()
    assert j == open(os.path.join(GOLDEN, "cfg1.json"), "rb").read()
    assert len(j) == 401
    # both parse back to the reference's data model
    doc = yaml.safe_load(y)
    assert doc == {"cdiVersion": "0.6.0", "kind": "nvidia.com/gpu", "devices": [
        {"name": "0", "annotations": {"attach-pci": "true", "bdf": "0000:c1:00.0", "cdi.k8s.io/vfio214": "nvidia.com/gpu=0"},
         "containerEdits": {"deviceNodes": [{"path": "/dev/vfio/214"}]}}]}
    jd = json.loads(j)
    assert jd["devices"] == doc["devices"] and jd["containerEdits"] == {}


def test_cdi_emit_vs_python(oracle, workloads):
    devs = workloads.cfg5_devices(3000)
    tup = [(d["bdf"].decode(), int(d["iommu_group"]), int(d["index"])) for d in devs]
    assert oracle.cdi_emit(1, devs) == pyref.cdi_json(tup)
    assert oracle.cdi_emit(0, devs) == pyref.cdi_yaml(tup)
    assert oracle.cdi_emit(0, devs[:0]) == pyref.cdi_yaml([]) == b"cdiVersion: 0.6.0\nkind: nvidia.com/gpu\ndevices: []\n"
    assert oracle.cdi_emit(1, devs[:0]) == pyref.cdi_json([])
    # YAML must parse back with string-typed bdf for quoted and plain forms alike (PyYAML 1.1
    # resolves sexagesimal ints, which is exactly why yaml.v3 quotes them)
    doc = yaml.safe_load(oracle.cdi_emit(0, devs[:600]))
    assert [d["annotations"]["bdf"] for d in doc["devices"]] == [t[0] for t in tup[:600]]


def test_base60_predicate(oracle):
    yes = [b"0000:41:00.0", b"0000:01:00.0", b"0000:59:19.7", b"0001:00:00.0", b"1:2", b"+1_0:59.", b"0:0:0"]
    no = [b"0000:c1:00.0", b"0000:3d:00.0", b"0000:65:00.0", b"0000:81:00.0", b"0000:59:1f.0", b"0000", b":1", b"1:", b"1:60",
          b"1:2:", b"1:2.3.4", b"a:1"]
    for s in yes:
        assert oracle.is_base60(s) and pyref.BASE60.match(s.decode())
    for s in no:
        assert not oracle.is_base60(s) and not pyref.BASE60.match(s.decode())


def test_full_size_cfg5_sizes(oracle, workloads):
    devs = workloads.cfg5_devices()
    j, y = oracle.cdi_emit(1, devs), oracle.cdi_emit(0, devs)
    assert len(j) == 20585718            # SURVEY.md 8(a) A12
    assert len(y) == 13330372
    names, offs = oracle.alloc_names(devs["index"])
    assert names[:16] == b"nvidia.com/gpu=0" and names.endswith(b"nvidia.com/gpu=65535") and offs[-1] == len(names)


def _rec_dicts(recs):
    out = []
    for r in recs:
        fl = int(r["flags"])
        out.append(dict(bdf=r["bdf"], is_dir=bool(fl & 16),
                        vendor=None if fl & 1 else bytes(r["vendor_txt"][:r["vendor_len"]]),
                        device=None if fl & 8 else bytes(r["device_txt"][:r["device_len"]]),
                        driver=None if fl & 2 else r["driver"], group=None if fl & 4 else int(r["iommu_group"])))
    return out


def check_classify(res, recs):
    iommu, devmap, accept = pyref.classify(_rec_dicts(recs))
    want_acc = np.array([0xFFFFFFFF if a is None else a for a in accept], dtype=np.uint32)
    assert np.array_equal(res["accept_index"], want_acc)
    assert res["n_accepted"] == sum(a is not None for a in accept)
    assert list(res["group_ids"]) == list(iommu.keys())
    for gi, g in enumerate(iommu):
        mem = res["group_members"][res["group_off"][gi]:res["group_off"][gi + 1]]
        assert [(recs["bdf"][m], int(res["accept_index"][m])) for m in mem] == iommu[g]
    assert [int(x).to_bytes(8, "little").rstrip(b"\0") for x in res["dev_ids"]] == list(devmap.keys())
    for di, d in enumerate(devmap):
        assert list(res["dev_groups"][res["dev_off"][di]:res["dev_off"][di + 1]]) == devmap[d]


def test_classify_cfg1(oracle, workloads):
    res = oracle.classify(workloads.cfg1_record())
    assert list(res["accept_index"]) == [0] and list(res["group_ids"]) == [214]
    assert res["dev_ids"][0] == int.from_bytes(b"2330", "little") and list(res["dev_groups"]) == [214]


def test_classify_vs_python(oracle, workloads, oracle_rows):
    recs = workloads.cfg3_records(oracle_rows["key"], n=5000, seed=3)
    rng = np.random.default_rng(5)
    # stress the edge cases: shuffled groups, unreadable files, directories, odd vendor text
    recs["iommu_group"] = rng.integers(0, 300, len(recs)).astype(np.uint32)
    recs["flags"] |= np.where(rng.random(len(recs)) < 0.05, 8, 0).astype(np.uint8)   # device read error
    recs["flags"] |= np.where(rng.random(len(recs)) < 0.02, 4, 0).astype(np.uint8)   # iommu link error
    recs["flags"] |= np.where(rng.random(len(recs)) < 0.02, 1, 0).astype(np.uint8)   # vendor read error
    recs["flags"] |= np.where(rng.random(len(recs)) < 0.01, 16, 0).astype(np.uint8)  # directory
    odd = rng.random(len(recs)) < 0.02
    recs["vendor_txt"][odd] = np.frombuffer(b"0x10DE\n\0", np.uint8)
    check_classify(oracle.classify(recs), recs)


def test_lw_encode(oracle):
    b = oracle.lw_encode(np.array([214, 7], np.uint32), np.array([1, 0], np.uint8))
    assert b == (b"\x0a\x0e\x0a\x03214\x12\x07Healthy" + b"\x0a\x0e\x0a\x017\x12\x09Unhealthy")


def test_all_threads_single_pass_equals_sequential(oracle, pci_text):
    """kxo_table_build_mt (the all-cores CPU comparator of bench.py: shards cut at vendor lines, first
    anchors min-merged) == kxo_table_build on the whole text, incl. duplicates across shards and a
    >= 64 KiB line in a middle shard."""
    texts = [pci_text, pci_text * 3, pci_text[700000:pci_text.find(b"\n", 1400000) + 1] + pci_text, b"", b"\tx\n",
             b"1111  one\n\t0001  a\n" * 300 + b"3333  " + b"x" * 70000 + b"\n\t0003  hidden\n" + b"4444  f\n\t0004  h\n" * 300]
    for t in texts:
        want = oracle.table_build(t)
        for th in (1, 2, 3, 8, 33):
            got = oracle.table_build_mt(t, th)
            assert np.array_equal(want, got), (len(t), th)
    dt, ps, offs = oracle.bench_parse_mt(pci_text * 2, oracle.table_build(pci_text)["key"][:500], 4)
    assert np.array_equal(offs, oracle.table_build(pci_text)["line_off"][:500].astype(np.int64)) and 0 < ps <= dt
