"""CPU tests of the host gathers under Plugin::pcieTopologyAware on nested fake sysfs trees: the walk and the fast gather
(1 and 4 threads) read each entry's link once, cut it at the first "pci" component, store targets over 120 bytes and
failed reads as unknown, and with the setting off read nothing and return the same records."""
import numpy as np
import pytest

import fake_sysfs
import pcie_host
from oracle import oracle as O

NV = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
LONG = "pci0000:00/" + "/".join("0000:%02x:00.0" % k for k in range(1, 10)) + "/0000:0a:00.0"
DEVS = [
    dict(bdf="0000:03:00.0", path="pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.0", group=10, **NV),
    dict(bdf="0000:04:00.0", path="pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:01.0/0000:04:00.0", group=11, **NV),
    dict(bdf="0000:05:00.0", path="platform/0000:05:00.0", group=12, **NV),                       # no pci component
    dict(bdf="0000:0a:00.0", path=LONG, group=13, **NV),                                        # 10 components, 126 bytes
    dict(bdf="0000:0b:00.0", path="pci10000:e0/10000:e0:1d.0/0000:0b:00.0", group=14, vendor=b"0x8086\n",
         device=b"0x1234\n", driver="ixgbe"),                                                   # not a candidate: still read
    dict(bdf="0000:0c:00.0", path=None, group=15, **NV),                                        # a plain directory
]


def _want(d):
    if d["path"] is None or not d["path"].startswith("pci") or len(d["path"]) > 120:
        return b"", 0
    return d["path"].encode(), len(d["path"])


@pytest.mark.parametrize("relative", [False, True])
@pytest.mark.parametrize("mode", [("walk", 0), ("fast", 1), ("fast", 4)])
def test_gather_paths(tmp_path, relative, mode):
    base = pcie_host.make_nested_tree(str(tmp_path), DEVS, relative=relative)
    assert len(LONG) > 120
    recs, paths, _ = pcie_host.gather(base, O.DEVREC_DTYPE, True, fast=mode[0] == "fast", threads=mode[1])
    assert len(paths) == len(recs)
    by_bdf = {bytes(r["bdf"]): p for r, p in zip(recs, paths)}
    for d in DEVS:
        if d["path"] is None:
            continue
        p = by_bdf[d["bdf"].encode()]
        want, n = _want(d)
        assert (bytes(p["path"]), int(p["len"])) == (want, n), d["bdf"]
    # the plain directory is walked into: its records have no path (readlink fails on a file)
    inner = [p for r, p in zip(recs, paths) if bytes(r["bdf"]) in (b"vendor", b"device", b"driver", b"iommu_group")]
    assert inner and all(int(p["len"]) == 0 for p in inner)
    # the records themselves are the ones the setting-off gather returns
    assert recs.tobytes() == fake_sysfs.gather(base, O.DEVREC_DTYPE).tobytes()


@pytest.mark.parametrize("fast", [False, True])
def test_setting_off_reads_nothing(tmp_path, fast):
    base = pcie_host.make_nested_tree(str(tmp_path), DEVS)
    recs, paths, reads = pcie_host.gather(base, O.DEVREC_DTYPE, False, fast=fast, count=True)
    assert reads == 0 and len(paths) == 0
    assert recs.tobytes() == fake_sysfs.gather(base, O.DEVREC_DTYPE).tobytes()
    recs_on, paths_on, reads_on = pcie_host.gather(base, O.DEVREC_DTYPE, True, fast=fast, count=True)
    assert reads_on == len(recs_on) == len(paths_on) and recs_on.tobytes() == recs.tobytes()
    # the seam's answers are the default read's
    _, fast_paths, _ = pcie_host.gather(base, O.DEVREC_DTYPE, True, fast=True, threads=4)
    assert np.array_equal(paths_on, fast_paths)
