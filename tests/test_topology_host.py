"""CPU tests of the host plugin's NUMA read (Plugin::topologyAware): gathered records byte for byte on fake trees for
every numa_node case of include/kxpu.h, through the walk, the fast gather at 1 and N threads and the mdev gather; with
topologyAware off the records are unchanged and no numa_node is opened."""
import os

import numpy as np
import pytest

import fake_mdev
import fake_sysfs
import topo_host
from oracle.mdev_oracle import MDEVREC_DTYPE
from oracle.oracle import DEVREC_DTYPE

# numa_node file contents -> the node the record must carry (None: unknown, no KXPU_REC_NUMA)
CASES = [(b"0\n", 0), (b"1\n", 1), (b"63\n", 63), (b"7", 7), (b"-1\n", None), (b"64\n", None), (b"99\n", None),
         (b"01\n", None), (b"\n", None), (b"", None), (b"junk\n", None), (b"1\n\n", None), (b" 1\n", None),
         (b"+1\n", None), (b"100\n", None), (None, None)]


def _tree(tmp_path):
    devs, numa, want = [], {}, {}
    for i, (raw, node) in enumerate(CASES):
        bdf = "0000:%02x:00.0" % (i + 1)
        devs.append(dict(bdf=bdf, vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=10 + i))
        if raw is not None:
            numa[bdf] = raw
        want[bdf] = node
    # records the walk stops early on: their numa_node is never read
    devs.append(dict(bdf="0000:80:00.0", vendor=b"0x8086\n", device=b"0x1234\n", driver="vfio-pci", group=90))
    devs.append(dict(bdf="0000:81:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="nvidia", group=91))
    devs.append(dict(bdf="0000:82:00.0", vendor=b"0x10de\n", device=None, driver="vfio-pci", group=92))  # device read fails
    for bdf in ("0000:80:00.0", "0000:81:00.0", "0000:82:00.0"):
        numa[bdf] = b"1\n"
    want["0000:82:00.0"] = 1  # a device-read failure still reaches the end of the record
    base = fake_sysfs.make_tree(str(tmp_path), devs)
    topo_host.add_numa(str(tmp_path), numa)
    return base, want


def _expect(plain, want):
    exp = plain.copy()
    for r in exp:
        node = want.get(r["bdf"].decode())
        if node is not None:
            r["flags"] |= 64
            r["reserved0"] = node
    return exp


def test_walk_records_every_numa_case(tmp_path):
    base, want = _tree(tmp_path)
    plain, reads0 = topo_host.gather(base, DEVREC_DTYPE, topo=False)
    assert reads0 == 0  # topologyAware off: numa_node is never opened
    assert plain.tobytes() == fake_sysfs.gather(base, DEVREC_DTYPE).tobytes()  # and the records are today's
    assert not (plain["flags"] & 64).any() and not plain["reserved0"].any()
    got, reads = topo_host.gather(base, DEVREC_DTYPE, topo=True)
    assert got.tobytes() == _expect(plain, want).tobytes()
    assert reads == len(CASES) + 1  # every record that reached its device read, nothing else


@pytest.mark.parametrize("threads", [1, 4])
def test_fast_gather_records_every_numa_case(tmp_path, threads):
    base, want = _tree(tmp_path)
    plain = fake_sysfs.gather(base, DEVREC_DTYPE)
    off, reads0 = topo_host.gather(base, DEVREC_DTYPE, topo=False, fast=True, threads=threads)
    assert reads0 == 0 and off.tobytes() == fake_sysfs.gather_fast(base, DEVREC_DTYPE, threads).tobytes() == plain.tobytes()
    # the default seam: the fast gather reads numa_node with openat on its own directory descriptor
    got, _ = topo_host.gather(base, DEVREC_DTYPE, topo=True, fast=True, threads=threads, count=False)
    assert got.tobytes() == _expect(plain, want).tobytes()


def test_fast_gather_many_entries_threads(tmp_path):
    devs, numa, want = [], {}, {}
    for i in range(300):
        bdf = "0000:%02x:%02x.%d" % (i >> 8, (i >> 3) & 31, i & 7)
        devs.append(dict(bdf=bdf, vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=i >> 3))
        raw, node = CASES[i % len(CASES)]
        if raw is not None:
            numa[bdf] = raw
        want[bdf] = node
    base = fake_sysfs.make_tree(str(tmp_path), devs)
    topo_host.add_numa(str(tmp_path), numa)
    plain = fake_sysfs.gather(base, DEVREC_DTYPE)
    walk, _ = topo_host.gather(base, DEVREC_DTYPE, topo=True)
    for t in (1, 4):
        fast, _ = topo_host.gather(base, DEVREC_DTYPE, topo=True, fast=True, threads=t, count=False)
        assert fast.tobytes() == walk.tobytes() == _expect(plain, want).tobytes()


def test_mdev_records_carry_the_parents_node(tmp_path):
    root = str(tmp_path)
    parents = {}
    mdevs, want = [], {}
    for i, (raw, node) in enumerate(CASES):
        parent = "0000:%02x:00.0" % (i + 1)
        parents[parent] = b"0x10de\n"
        u = "%08x-0000-4000-8000-%012x" % (i, i)
        mdevs.append(dict(uuid=u, parent=parent, group=300 + i))
        want[u] = node
    # a record without a type name still reads its node (it may join an existing group)
    mdevs.append(dict(uuid="%08x-0000-4000-8000-%012x" % (99, 99), parent="0000:01:00.0", group=300, name=None))
    want[mdevs[-1]["uuid"]] = 0
    mbase = fake_mdev.make_tree(root, mdevs, parents=parents)
    topo_host.add_numa(root, {"0000:%02x:00.0" % (i + 1): raw for i, (raw, _) in enumerate(CASES) if raw is not None})
    classes = [("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-vgpu")]
    plain, reads0 = topo_host.gather_mdev(mbase, classes, MDEVREC_DTYPE, topo=False)
    assert reads0 == 0 and plain.tobytes() == fake_mdev.gather(mbase, classes).tobytes()
    got, reads = topo_host.gather_mdev(mbase, classes, MDEVREC_DTYPE, topo=True)
    exp = plain.copy()
    for r in exp:
        node = want.get(r["uuid"].decode())
        if node is not None:
            r["flags"] |= 64
            r["reserved0"] = node
    assert got.tobytes() == exp.tobytes()
    assert reads == len(mdevs)


def test_options_and_preferred_allocation_off(tmp_path):
    """topologyAware off: the reference's options and its empty GetPreferredAllocation answer (no GPU call)."""
    hp = fake_sysfs.HostPlugin.__new__(fake_sysfs.HostPlugin)
    hp.L = fake_sysfs.host_lib()
    hp.h = hp.L.kxh_new(None, str(tmp_path).encode(), b"/nonexistent", str(tmp_path).encode())
    try:
        assert topo_host.options(hp) == dict(PreStartRequired=False, GetPreferredAllocationAvailable=False)
        idx = hp.L.kxh_add_plugin(hp.h, b"GPU", str(tmp_path).encode(), b"1,2,3")
        assert topo_host.preferred_allocation(hp, idx, [(["1", "2", "3"], ["1"], 2)]) == []
        topo_host.set_topology(hp, True)
        assert topo_host.options(hp) == dict(PreStartRequired=False, GetPreferredAllocationAvailable=True)
        with pytest.raises(RuntimeError, match="unknown device: 7"):
            topo_host.preferred_allocation(hp, idx, [(["1", "7"], [], 1)])
    finally:
        hp.close()
