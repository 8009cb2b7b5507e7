"""Records for the IOMMU group viability tests (kxpu_classify_viable, ABI v8): a record builder, the hand cases and a
hypothesis strategy, shared by the CPU and the GPU tests."""
import numpy as np
from hypothesis import strategies as st

from oracle import xpu_oracle as XO

NV = [(b"10de", b"vfio-pci")]
TWO = [(b"10de", b"vfio-pci"), (b"1002", b"vfio-pci")]
BLOCKS, IS_DIR, VENDOR_ERR, DRIVER_ERR, IOMMU_ERR, DEVICE_ERR, NUMA = 0x80, 0x10, 0x01, 0x02, 0x04, 0x08, 0x40
VIABLE = 0xFFFFFFFF


def rec(bdf, group, driver=b"vfio-pci", vendor=b"0x10de\n", device=b"0x2330\n", flags=0, numa=0):
    r = np.zeros(1, XO.DEVREC_DTYPE)[0]
    r["bdf"] = bdf
    r["vendor_txt"][:len(vendor)] = np.frombuffer(vendor, np.uint8)
    r["vendor_len"] = len(vendor)
    r["device_txt"][:len(device)] = np.frombuffer(device, np.uint8)
    r["device_len"] = len(device)
    r["driver"] = driver
    r["iommu_group"] = group
    r["flags"] = flags
    r["reserved0"] = numa
    return r


def gpu(i, group, **kw):
    return rec(b"0000:%02x:00.0" % i, group, **kw)


def audio(i, group, driver=b"snd_hda_intel"):
    return rec(b"0000:%02x:00.1" % i, group, driver=driver, device=b"0x22a3\n", flags=BLOCKS)


def host(i, group, driver=b"nvme", vendor=b"0x144d\n"):
    return rec(b"0000:%02x:00.2" % i, group, driver=driver, vendor=vendor, device=b"0xa80a\n", flags=BLOCKS)


def arr(*rs):
    return np.array(list(rs), XO.DEVREC_DTYPE)


# name -> (records, [(group id, first blocker)] in group ordinal order)
HAND = {
    "blocker_after_first_member": (arr(gpu(1, 7), audio(1, 7)), [(7, 1)]),
    "blocker_before_first_member": (arr(host(0, 7), gpu(1, 7), gpu(2, 8)), [(7, 0), (8, VIABLE)]),
    "several_blockers_min_wins": (arr(gpu(0, 9), host(1, 5), audio(2, 9), host(3, 9), gpu(4, 5), host(5, 5)),
                                  [(9, 2), (5, 1)]),
    "blocker_only_group": (arr(host(0, 3), host(1, 3), gpu(2, 4)), [(4, VIABLE)]),
    "group_whose_only_candidate_has_device_err": (arr(gpu(0, 6, flags=DEVICE_ERR), audio(0, 6), gpu(1, 2)),
                                                  [(2, VIABLE)]),
    "blocks_on_a_candidate_is_ignored": (arr(gpu(0, 1, flags=BLOCKS), gpu(1, 1, flags=BLOCKS)), [(1, VIABLE)]),
    "blocks_on_a_directory_is_ignored": (arr(rec(b"0000:00:00.0", 1, driver=b"", flags=IS_DIR | BLOCKS), gpu(1, 1)),
                                         [(1, VIABLE)]),
    "group_0": (arr(audio(0, 0), gpu(1, 0), host(2, 0)), [(0, 0)]),
    "unbound_and_allowed_functions_are_not_blockers": (
        arr(gpu(0, 4), rec(b"0000:00:00.1", 4, driver=b"", flags=DRIVER_ERR),
            rec(b"0000:00:00.2", 4, driver=b"pcieport", vendor=b"0x10b5\n"),
            rec(b"0000:00:00.3", 4, driver=b"pci-stub", device=b"0x22a3\n")), [(4, VIABLE)]),
    "blocks_with_a_failed_read_still_blocks": (arr(gpu(0, 4), rec(b"0000:00:00.1", 4, driver=b"", flags=DRIVER_ERR | BLOCKS)),
                                               [(4, 1)]),
    "n_0": (arr(), []),
}


@st.composite
def viab_recs(draw):
    """Up to 48 records over 8 groups: GPUs (some with failed reads), audio / host functions with and without the flag,
    directories, flags on candidates, the NUMA flag; topology-relevant and irrelevant bits mixed freely."""
    n = draw(st.integers(0, 48))
    out = np.zeros(n, XO.DEVREC_DTYPE)
    for i in range(n):
        g = draw(st.integers(0, 7))
        kind = draw(st.sampled_from(["gpu", "gpu", "amd", "audio", "host", "port"]))
        if kind == "gpu":
            r = gpu(i, g, device=draw(st.sampled_from([b"0x2330\n", b"0x2331\n"])))
        elif kind == "amd":
            r = rec(b"0000:%02x:00.0" % i, g, vendor=b"0x1002\n", device=b"0x740f\n")
        elif kind == "audio":
            r = audio(i, g, driver=draw(st.sampled_from([b"snd_hda_intel", b"vfio-pci"])))
        elif kind == "host":
            r = host(i, g)
        else:
            r = rec(b"0000:%02x:00.0" % i, g, driver=b"pcieport", vendor=b"0x10b5\n")
        fl = int(r["flags"])
        for bit in (BLOCKS, IS_DIR, VENDOR_ERR, DRIVER_ERR, IOMMU_ERR, DEVICE_ERR):
            if draw(st.integers(0, 9)) == 0:
                fl ^= bit
        if draw(st.booleans()):
            fl |= NUMA
            r["reserved0"] = draw(st.integers(0, 3))
        r["flags"] = fl
        out[i] = r
    return out
