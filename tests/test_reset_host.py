"""CPU tests of the host plugin's reset reads (Plugin::resetCheck) on fake sysfs trees with reset_method and reset files:
what each gather stores for candidates, class-bound and foreign functions, the read-error and legacy flags, no reset file
opened with the setting off, and the start-up refusals of resetMethods."""
import os

import pytest

import dra_host as DH
import fake_sysfs
import pcie_host
import reset_host as H
from kxpu_b200.binding import RS_ABSENT, RS_LEGACY, RS_READ_ERR
from oracle import xpu_oracle as XO

NVD = dict(vendor=b"0x10de\n", device=b"0x2330\n")
SW = "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:08.0"
DEVS = [dict(bdf="0000:03:00.0", group=30, driver="vfio-pci", path=SW + "/0000:03:00.0", **NVD),   # FLR
        dict(bdf="0000:03:00.1", group=30, driver="snd_hda_intel", path=SW + "/0000:03:00.1", vendor=b"0x10de\n",
             device=b"0x22a3\n"),                                                                     # same vendor
        dict(bdf="0000:03:00.2", group=31, driver="vfio-pci", path=SW + "/0000:03:00.2", vendor=b"0x1b21\n",
             device=b"0x1242\n"),                                                                     # foreign, on vfio
        dict(bdf="0000:05:00.0", group=50, driver="vfio-pci", path="pci0000:00/0000:05:00.0", **NVD),  # legacy kernel
        dict(bdf="0000:06:00.0", group=60, driver="nvme", path="pci0000:00/0000:00:02.0/0000:06:00.0",
             vendor=b"0x144d\n", device=b"0xa80a\n"),
        dict(bdf="0000:07:00.0", group=70, path="pci0000:00/0000:00:03.0/0000:07:00.0", **NVD)]     # unbound


@pytest.fixture
def tree(tmp_path):
    base = pcie_host.make_nested_tree(str(tmp_path), DEVS, relative=True)
    H.set_method(base, "0000:03:00.0", b"flr bus\n")
    H.set_method(base, "0000:03:00.1", b"flr\n")   # no candidate: never read
    H.set_method(base, "0000:05:00.0", None, legacy=True)
    H.set_method(base, "0000:06:00.0", b"flr\n")
    return str(tmp_path), base


def _by_bdf(recs, *cols):
    return {bytes(r["bdf"]).rstrip(b"\0").decode(): tuple(c[i] for c in cols) for i, r in enumerate(recs)}


@pytest.mark.parametrize("fast", [False, True])
def test_reads_of_the_walk(tree, fast):
    _, base = tree
    recs, paths, rrs, reads = H.gather(base, XO.DEVREC_DTYPE, True, fast=fast)
    assert reads == 3  # reset_method of the two candidates, and reset where reset_method is missing
    got = _by_bdf(recs, recs, paths, rrs)
    r, p, s = got["0000:03:00.0"]
    assert bytes(s["txt"][:s["len"]]) == b"flr bus\n" and s["flags"] == 0
    assert bytes(p["path"])[:p["len"]] == (SW + "/0000:03:00.0").encode()
    assert got["0000:05:00.0"][2]["flags"] == RS_ABSENT | RS_LEGACY
    for bdf in ("0000:03:00.1", "0000:03:00.2", "0000:06:00.0", "0000:07:00.0"):  # no candidates: no reset read
        assert got[bdf][2].tobytes() == bytes(80)
    # every entry's driver, and the group of one bound to a class driver, for the bus-reset sets
    assert bytes(got["0000:03:00.1"][0]["driver"]).rstrip(b"\0") == b"snd_hda_intel"
    assert bytes(got["0000:06:00.0"][0]["driver"]).rstrip(b"\0") == b"nvme"
    assert bytes(got["0000:03:00.2"][0]["driver"]).rstrip(b"\0") == b"vfio-pci"
    assert int(got["0000:03:00.2"][0]["iommu_group"]) == 31
    assert int(got["0000:07:00.0"][0]["flags"]) & 0x02  # unbound: the class test's driver error stays
    # with the setting off: no reset file opened, no path read, and the candidates' records are the same bytes
    recs_off, paths_off, rrs_off, reads_off = H.gather(base, XO.DEVREC_DTYPE, False, fast=fast)
    assert reads_off == 0 and rrs_off.tobytes() == bytes(80 * len(rrs_off)) and paths_off.tobytes() == bytes(128 * len(paths_off))
    for a, b in zip(recs_off, recs):
        if bytes(a["driver"]).rstrip(b"\0") in (b"vfio-pci",) and bytes(a["vendor_txt"][:7]) == b"0x10de\n":
            assert a.tobytes() == b.tobytes()


def test_read_flags(tree):
    _, base = tree
    H.set_method(base, "0000:05:00.0", None)  # a kernel of 5.15 or later with no method: neither file
    d = os.path.realpath(os.path.join(base, "0000:03:00.0"))
    os.remove(os.path.join(d, "reset_method"))
    os.mkdir(os.path.join(d, "reset_method"))  # reading a directory fails with EISDIR: a read error
    H.set_method(base, "0000:07:00.0", b"x" * 100)
    recs, _, rrs, reads = H.gather(base, XO.DEVREC_DTYPE, True)
    got = _by_bdf(recs, rrs)
    assert got["0000:05:00.0"][0]["flags"] == RS_ABSENT
    assert got["0000:03:00.0"][0]["flags"] == RS_READ_ERR
    assert reads == 3


def test_over_long_file(tree):
    _, base = tree
    H.set_method(base, "0000:03:00.0", b"flr " * 40)
    recs, _, rrs, _ = H.gather(base, XO.DEVREC_DTYPE, True)
    s = _by_bdf(recs, rrs)["0000:03:00.0"][0]
    assert s["len"] == 65 and bytes(s["txt"]) == (b"flr " * 40)[:64]


@pytest.fixture
def hp(tree, tmp_path):
    p = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), tree[1], str(tmp_path / "pci.ids"), str(tmp_path) + "/")
    try:
        yield p
    finally:
        p.close()


@pytest.mark.parametrize("methods,why", [
    (["flr", "warm"], "resetMethods: warm is not a reset method (flr, af_flr, pm, bus, cxl_bus, device_specific, acpi)"),
    (["flr", "pm", "flr"], "resetMethods: flr is listed twice"),
    (["FLR"], "resetMethods: FLR is not a reset method (flr, af_flr, pm, bus, cxl_bus, device_specific, acpi)"),
])
def test_start_up_refusals(hp, methods, why):
    H.set_reset(hp, True, methods)
    assert DH.initiate(hp) == why
    assert H.reads(hp) == 0
