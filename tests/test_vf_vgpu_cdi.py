"""CPU checks of the typed VF-vGPU CDI layouts (kxpu_cdi_emit_vf_vgpu[_cdev]): the C oracle (tests/vf_vgpu_cdi_oracle.c)
against the Python restatement (tests/pyref_vf_vgpu_cdi.py), over edge IDs, keys that would resolve as non-strings if
written plain, base-60 quoted and plain bdfs, both formats and both node layouts, and a hypothesis strategy over all of
them.  Every annotation reads back with PyYAML / json as the string it was written from, and without the two new
annotations the document is the C oracle's kxpu_cdi_emit_kind document (group layout) of the same records."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import cdev_cases as CC
import pyref_vf_vgpu_cdi as PV
import vf_vgpu_cdi_cases as K
import vf_vgpu_cdi_oracle as VO
from kxpu_b200.binding import CDEV_FIELD, VFVGPUCDI_DTYPE
from oracle import xpu_oracle as XO

FORMATS = [K.FMT_YAML, K.FMT_JSON]


def _check(fmt, kind, recs, cdev):
    want = VO.emit(fmt, kind, recs, cdev)
    assert want == PV.emit(fmt, kind, recs, cdev)
    if want is None:
        return None
    anns = PV.annotations(fmt, want)
    assert len(anns) == len(recs)
    for a, r in zip(anns, recs):
        d = r["dev"]
        assert a == {"attach-pci": "true", "bdf": bytes(d["bdf"]).decode(),
                     "cdi.k8s.io/vfio%d" % d["iommu_group"]: "%s=%d" % (kind.decode(), d["index"]),
                     "vgpu-type": str(int(r["type_id"])), "vgpu-type-key": bytes(r["key"])[:int(r["key_len"])].decode()}
        assert all(type(v) is str for v in a.values())
    plain = CC.oracle_doc(fmt, kind, recs["dev"]) if cdev else XO.cdi_emit_kind(fmt, kind, recs["dev"])
    assert PV.strip_types(fmt, want) == plain
    return want


@pytest.mark.parametrize("cdev", [False, True])
@pytest.mark.parametrize("kind", K.KINDS)
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("n", [0, 1, 2, 17, 300])
def test_oracle_matches_restatement(fmt, kind, cdev, n):
    recs = K.records(n, seed=n)
    doc = _check(fmt, kind, recs, cdev)
    assert doc is not None
    if n == 0:  # the zero-device document is every layout's
        assert doc == XO.cdi_emit_kind(fmt, kind, recs["dev"])


@pytest.mark.parametrize("fmt", FORMATS)
def test_edge_values_are_quoted_strings(fmt):
    recs = K.records(len(K.EDGE_KEYS), seed=3)
    assert set(int(x) for x in recs["type_id"][:len(K.EDGE_IDS)]) == set(K.EDGE_IDS)
    doc = _check(fmt, K.KIND_14, recs, False)
    for key in K.TRICKY_KEYS:
        assert b'vgpu-type-key: "%s"\n' % key in doc if fmt == K.FMT_YAML else b'"vgpu-type-key": "%s"\n' % key in doc
    assert (b'vgpu-type: "4294967295"' if fmt == K.FMT_YAML else b'"vgpu-type": "4294967295"') in doc
    if fmt == K.FMT_YAML:  # both forms of the bdf: quoted where yaml.v3 would read base 60, plain elsewhere
        assert b'bdf: "0000:' in doc and b"bdf: 0000:" in doc


@pytest.mark.parametrize("cdev", [False, True])
@pytest.mark.parametrize("fmt", FORMATS)
def test_domain(fmt, cdev):
    good = K.records(3, seed=5)
    assert _check(fmt, K.KIND_14, good, cdev) is not None
    bad = []
    r = good.copy(); r["type_id"][1] = 0; bad.append(r)
    r = good.copy(); r["key_len"][1] = 0; bad.append(r)
    r = good.copy(); r["key_len"][1] = 41; bad.append(r)
    for c in (b" ", b"/", b'"', b":", b"\xff", b"\x00"):
        r = good.copy(); key = bytearray(bytes(r["key"][2]).ljust(40, b"x")); key[0:1] = c
        r["key"][2] = bytes(key); r["key_len"][2] = 3; bad.append(r)
    r = good.copy(); r["dev"]["bdf"][0] = b"0000:C1:00.0"; bad.append(r)
    for r in bad:
        assert VO.emit(fmt, K.KIND_14, r, cdev) is None and PV.emit(fmt, K.KIND_14, r, cdev) is None
    assert VO.emit(fmt, b"nvidia.com", good, cdev) is None and PV.emit(fmt, b"nvidia.com", good, cdev) is None


_KEY = st.one_of(st.sampled_from(K.TRICKY_KEYS),
                 st.text(alphabet="ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_.-", min_size=1,
                         max_size=40).map(str.encode))
_BDF = st.builds(lambda d, b, s, f: b"%04x:%02x:%02x.%d" % (d, b, s, f), st.integers(0, 0xFFFF), st.integers(0, 255),
                 st.integers(0, 31), st.integers(0, 7))
_DEV = st.tuples(_BDF, st.integers(0, (1 << 32) - 1), st.integers(0, (1 << 32) - 1), st.integers(0, (1 << 64) - 1),
                 st.integers(1, (1 << 32) - 1), _KEY)


@settings(max_examples=150, deadline=None)
@given(devs=st.lists(_DEV, max_size=6, unique_by=lambda d: d[3]), fmt=st.sampled_from(FORMATS), cdev=st.booleans(),
       kind=st.sampled_from(K.KINDS))
def test_hypothesis(devs, fmt, cdev, kind):
    recs = np.zeros(len(devs), VFVGPUCDI_DTYPE)
    for i, (bdf, group, node, index, tid, key) in enumerate(devs):
        recs[i]["dev"]["bdf"], recs[i]["dev"]["iommu_group"], recs[i]["dev"][CDEV_FIELD] = bdf, group, node
        recs[i]["dev"]["index"], recs[i]["type_id"], recs[i]["key"], recs[i]["key_len"] = index, tid, key, len(key)
    assert _check(fmt, kind, recs, cdev) is not None
