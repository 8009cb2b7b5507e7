"""CPU checks of the vGPU cdev CDI spec (kxpu_cdi_emit_mdev_cdev / kxpu_cdi_parse_mdev_cdev, additions to ABI v14): the
Python restatement (pyref_mdev_cdev) against the document derived from the C oracle, pyref_mdev_cdev's parse verdicts,
the four layouts against each other, and the ABI surface."""
import os
import re

import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import mdev_cdev_cases as K
import pyref_cdev as PC
import pyref_cdi_parse as PP
import pyref_mdev_cdev as PMC
from conftest import ROOT
from oracle import mdev_oracle as MO
from oracle import xpu_oracle as XO

FMTS = [K.FMT_YAML, K.FMT_JSON]
KINDS = [K.KIND_SHORT, K.KIND_LONG]


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [0, 1, 4, 300])
def test_restatement_equals_oracle(fmt, kind, n):
    recs = K.records(n, seed=n + 3)
    want = K.oracle_doc(fmt, kind, recs)
    assert PMC.emit(fmt, kind, recs) == want
    if n >= 4:
        assert b"/dev/vfio/devices/vfio4294967295" in want
    assert b"/dev/iommu" not in want


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("node", K.EDGE_N)
def test_one_device_per_edge_number(fmt, kind, node):
    recs = K.records(1, seed=5)
    recs["vfio_cdev"] = node
    doc = PMC.emit(fmt, kind, recs)
    assert doc == K.oracle_doc(fmt, kind, recs)
    assert PMC.node_path(node) in doc


@settings(max_examples=200, deadline=None)
@given(n=st.integers(0, 12), seed=st.integers(0, 2 ** 31), fmt=st.sampled_from(FMTS), kind=st.sampled_from(KINDS),
       nodes=st.lists(st.integers(0, (1 << 32) - 1), min_size=12, max_size=12))
def test_restatement_equals_oracle_fuzz(n, seed, fmt, kind, nodes):
    recs = K.records(n, seed)
    recs["vfio_cdev"] = nodes[:n]
    assert PMC.emit(fmt, kind, recs) == K.oracle_doc(fmt, kind, recs)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", KINDS)
def test_only_the_node_differs_from_the_mdev_layout(fmt, kind):
    """Annotations (mdev included), head, tail and the zero-device form are the vGPU group layout's; the node names N."""
    recs = K.records(50, seed=9)
    group_doc, cdev_doc = MO.cdi_emit_mdev(fmt, kind, np.ascontiguousarray(recs["dev"])), PMC.emit(fmt, kind, recs)
    assert K.swap_back(fmt, cdev_doc, recs) == group_doc
    nodes = [int(x) for x in re.findall(rb"/dev/vfio/devices/vfio(\d+)", cdev_doc)]
    assert nodes == [int(x) for x in recs["vfio_cdev"]]
    assert PMC.emit(fmt, kind, recs[:0]) == MO.cdi_emit_mdev(fmt, kind, np.ascontiguousarray(recs["dev"][:0]))


def test_refusals():
    recs = K.records(2)
    assert PMC.emit(K.FMT_YAML, b"no-slash", recs) is None
    assert PMC.parse(K.FMT_YAML, K.oracle_doc(K.FMT_YAML, K.KIND_SHORT, recs), b"no-slash")[0] == PMC.E_UNSUPPORTED
    bad = recs.copy()
    bad["dev"]["uuid"][1] = bad["dev"]["uuid"][1].upper()
    assert PMC.emit(K.FMT_YAML, K.KIND_SHORT, bad) is None
    bad = recs.copy()
    bad["dev"]["parent"][1] = b""
    assert PMC.emit(K.FMT_JSON, K.KIND_SHORT, bad) is None


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", KINDS)
def test_parse_restatement(fmt, kind):
    recs, docs = K.damaged(fmt, kind)
    verdicts = {}
    for name, doc in docs:
        st_, got = PMC.parse(fmt, doc, kind)
        verdicts[name] = st_
        if st_ == PMC.OK:
            assert PMC.emit(fmt, kind, got) == doc, name
    assert verdicts["clean"] == PMC.OK and verdicts["zero_devices"] == PMC.OK
    assert PMC.parse(fmt, docs[0][1], kind)[1].tobytes() == recs.tobytes()
    for name in ("node_leading_zero", "node_past_u32", "node_empty", "node_is_group", "group_past_u32", "iommu_node",
                 "uuid_upper", "trailing_byte", "crlf", "empty"):
        assert verdicts[name] == PMC.E_INVALID, name
    assert sum(v == PMC.E_INVALID for v in verdicts.values()) > 100


@pytest.mark.parametrize("fmt", FMTS)
def test_layouts_refuse_each_other(fmt):
    """Each of the four layouts' documents is refused by the other three parsers; the zero-device document is all four."""
    recs = K.records(3, seed=2)
    pci = np.zeros(3, XO.CDIDEV_DTYPE)
    pci["bdf"], pci["iommu_group"], pci["index"] = recs["dev"]["parent"], recs["dev"]["iommu_group"], recs["dev"]["index"]
    pci[PC.CDEV_FIELD] = recs["vfio_cdev"]
    docs = {"pci": XO.cdi_emit_kind(fmt, K.KIND_SHORT, pci), "cdev": PC.emit(fmt, K.KIND_SHORT, pci),
            "mdev": MO.cdi_emit_mdev(fmt, K.KIND_SHORT, np.ascontiguousarray(recs["dev"])),
            "mdev_cdev": PMC.emit(fmt, K.KIND_SHORT, recs)}
    parsers = {"pci": lambda d: PP.parse(fmt, d, K.KIND_SHORT)[0], "cdev": lambda d: PC.parse(fmt, d, K.KIND_SHORT)[0],
               "mdev": lambda d: PP.parse(fmt, d, K.KIND_SHORT, mdev=True)[0],
               "mdev_cdev": lambda d: PMC.parse(fmt, d, K.KIND_SHORT)[0]}
    for dl, doc in docs.items():
        for pl, parse in parsers.items():
            assert parse(doc) == (PMC.OK if dl == pl else PMC.E_INVALID), (dl, pl)
    zero = PMC.emit(fmt, K.KIND_SHORT, recs[:0])
    assert zero == XO.cdi_emit_kind(fmt, K.KIND_SHORT, pci[:0])
    for parse in parsers.values():
        assert parse(zero) == PMC.OK


def test_record_layout_and_abi_surface():
    from kxpu_b200 import binding as B
    assert B.MDEVCDEV_DTYPE == K.MDEVCDEV_DTYPE
    assert B.MDEVCDEV_DTYPE.itemsize == 80 and B.MDEVCDEV_DTYPE.fields["vfio_cdev"][1] == 64
    assert B.MDEVCDEV_DTYPE.fields["dev"][0] == B.MDEVCDI_DTYPE
    hdr = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    assert "#define KXPU_ABI_VERSION 14" in hdr
    assert re.search(r"typedef struct kxpu_mdevcdev \{\s*kxpu_mdevcdi dev;", hdr)
    for name in ("kxpu_cdi_emit_mdev_cdev", "kxpu_cdi_parse_mdev_cdev"):
        assert name in B.ABI_SYMBOLS
        assert re.search(r"int32_t %s\(" % name, hdr)
    go = open(os.path.join(ROOT, "integration", "go", "kxpu_cgo.go")).read()
    assert "C.kxpu_cdi_emit_mdev_cdev(" in go and "C.kxpu_cdi_parse_mdev_cdev(" in go


def test_frag_min_bounds_mdev_cdev_documents():
    """The shortest mdev cdev fragment is longer than the shortest group fragment, so KXPU_CDI_FRAG_MIN bounds the count."""
    from kxpu_b200 import binding as B
    recs = K.records(64)
    recs["dev"]["parent"], recs["dev"]["index"], recs["dev"]["iommu_group"] = b"a", np.arange(64) % 10, 0  # plain in YAML
    recs["vfio_cdev"] = 0
    doc = PMC.emit(K.FMT_YAML, b"a/b", recs)
    assert len(doc) // B.CDI_FRAG_MIN >= 64
