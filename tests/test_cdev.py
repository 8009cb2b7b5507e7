"""CPU checks of the VFIO cdev CDI spec (kxpu_cdi_emit_cdev / kxpu_cdi_parse_cdev, ABI v14): the Python restatement
(pyref_cdev) against the document derived from the C oracle, pyref_cdev's parse verdicts, and the ABI surface."""
import os
import re

import numpy as np
import pytest

import cdev_cases as K
import pyref_cdev as PC
from conftest import ROOT

FMTS = [K.FMT_YAML, K.FMT_JSON]
KINDS = [K.KIND_SHORT, K.KIND_LONG]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [0, 1, 4, 300])
def test_restatement_equals_oracle(fmt, kind, n):
    recs = K.records(n, seed=n + 3)
    want = K.oracle_doc(fmt, kind, recs)
    assert PC.emit(fmt, kind, recs) == want
    if n >= 4:
        assert b"/dev/vfio/devices/vfio4294967295" in want
    assert b"/dev/iommu" not in want


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("node", K.EDGE_N)
def test_one_device_per_edge_number(fmt, kind, node):
    recs = K.records(1, seed=5)
    recs[K.CDEV_FIELD] = node
    doc = PC.emit(fmt, kind, recs)
    assert doc == K.oracle_doc(fmt, kind, recs)
    assert (b"/dev/vfio/devices/vfio%d" % node) in doc


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", KINDS)
def test_only_the_node_differs_from_the_group_layout(fmt, kind):
    """Annotations, head, tail and the zero-device form are the group layout's; the node names N, not g."""
    from oracle import xpu_oracle as XO
    recs = K.records(50, seed=9)
    group_doc, cdev_doc = XO.cdi_emit_kind(fmt, kind, recs), PC.emit(fmt, kind, recs)
    pat = re.compile(rb"/dev/vfio/(devices/vfio)?\d+")
    assert pat.sub(b"NODE", group_doc) == pat.sub(b"NODE", cdev_doc)
    nodes = [int(x) for x in re.findall(rb"/dev/vfio/devices/vfio(\d+)", cdev_doc)]
    assert nodes == [int(x) for x in recs[K.CDEV_FIELD]]
    assert PC.emit(fmt, kind, recs[:0]) == XO.cdi_emit_kind(fmt, kind, recs[:0])


def test_kind_outside_the_domain():
    recs = K.records(2)
    assert PC.emit(K.FMT_YAML, b"no-slash", recs) is None
    assert PC.parse(K.FMT_YAML, K.oracle_doc(K.FMT_YAML, K.KIND_SHORT, recs), b"no-slash")[0] == PC.E_UNSUPPORTED


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", KINDS)
def test_parse_restatement(fmt, kind):
    recs, docs = K.damaged(fmt, kind)
    verdicts = {}
    for name, doc in docs:
        st, got = PC.parse(fmt, doc, kind)
        verdicts[name] = st
        if st == PC.OK:
            assert PC.emit(fmt, kind, got) == doc, name
    assert verdicts["clean"] == PC.OK and verdicts["zero_devices"] == PC.OK
    assert PC.parse(fmt, docs[0][1], kind)[1].tobytes() == recs.tobytes()
    for name in ("node_leading_zero", "node_past_u32", "node_empty", "node_is_group", "group_past_u32", "iommu_node",
                 "trailing_byte", "crlf", "empty"):
        assert verdicts[name] == PC.E_INVALID, name
    assert sum(v == PC.E_INVALID for v in verdicts.values()) > 100


@pytest.mark.parametrize("fmt", FMTS)
def test_layouts_refuse_each_other(fmt):
    """A group-layout document is not a cdev document; the zero-device document is both."""
    from oracle import xpu_oracle as XO
    import pyref_cdi_parse as PP
    recs = K.records(3, seed=2)
    assert PC.parse(fmt, XO.cdi_emit_kind(fmt, K.KIND_SHORT, recs), K.KIND_SHORT)[0] == PC.E_INVALID
    assert PP.parse(fmt, PC.emit(fmt, K.KIND_SHORT, recs), K.KIND_SHORT)[0] == PP.E_INVALID
    assert PC.parse(fmt, XO.cdi_emit_kind(fmt, K.KIND_SHORT, recs[:0]), K.KIND_SHORT)[0] == PC.OK


def test_abi_v14_surface():
    from kxpu_b200 import binding as B
    hdr = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    assert "#define KXPU_ABI_VERSION 14" in hdr
    assert {"kxpu_cdi_emit_cdev", "kxpu_cdi_parse_cdev"} <= set(B.ABI_SYMBOLS)
    assert B.CDEV_FIELD == K.CDEV_FIELD and B.CDIDEV_DTYPE.fields[B.CDEV_FIELD][1] == 20
    assert re.search(r"uint32_t vfio_cdev;", hdr)
    go = open(os.path.join(ROOT, "integration", "go", "kxpu_cgo.go")).read()
    assert "C.kxpu_cdi_emit_cdev(" in go and "C.kxpu_cdi_parse_cdev(" in go


def test_frag_min_bounds_cdev_documents():
    """The shortest cdev fragment is longer than the group layout's, so KXPU_CDI_FRAG_MIN still bounds the count."""
    from kxpu_b200 import binding as B
    recs = np.zeros(64, K.records(0).dtype)
    recs["bdf"], recs["index"] = b"1", np.arange(64) % 10
    doc = PC.emit(K.FMT_YAML, b"a/b", recs)
    assert len(doc) // B.CDI_FRAG_MIN >= 64
