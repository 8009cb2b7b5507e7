"""Records for the SR-IOV tests (kxpu_sriov, kxpu_pcie_tree_sriov): side-record builders, the hand cases and hypothesis
strategies, shared by the CPU and the GPU tests."""
import numpy as np
from hypothesis import strategies as st

import viab_cases as VC
from oracle import xpu_oracle as XO
from kxpu_b200.binding import PCIPATH_DTYPE, SRIOVREC_DTYPE

NV = VC.NV
NO_PF = VIABLE = 0xFFFFFFFF
PHYSFN_ERR, NUMVFS_ERR = 0x01, 0x02


def sr(physfn=b"", numvfs=b"", flags=0):
    s = np.zeros(1, SRIOVREC_DTYPE)[0]
    s["physfn"] = physfn
    s["numvfs_txt"][:min(len(numvfs), 8)] = np.frombuffer(numvfs[:8], np.uint8)
    s["numvfs_len"] = min(len(numvfs), 9)
    s["flags"] = flags
    return s


def walk(*rows):
    """rows of (devrec, sriovrec) -> (recs, srs)."""
    return (np.array([r for r, _ in rows], XO.DEVREC_DTYPE), np.array([s for _, s in rows], SRIOVREC_DTYPE))


def fn(bdf, group, driver=b"vfio-pci", flags=0, physfn=b"", numvfs=b"", sflags=0):
    """(devrec, sriovrec) of one function: flags are the devrec's KXPU_REC_*, sflags the side record's KXPU_SR_*."""
    return VC.rec(bdf, group, driver=driver, flags=flags), sr(physfn, numvfs, sflags)


# name -> ((recs, srs), pf_of, numvfs, {group id: blocking record or VIABLE}) under the NVIDIA class
HAND = {
    "vfs_under_a_host_pf": (walk(fn(b"0000:03:00.0", 50, driver=b"nvidia"),
                                 fn(b"0000:03:00.4", 51, physfn=b"0000:03:00.0"),
                                 fn(b"0000:03:00.5", 52, physfn=b"0000:03:00.0")),
                            [NO_PF, 0, 0], [0, 0, 0], {51: VIABLE, 52: VIABLE}),
    "pf_on_vfio_with_vfs": (walk(fn(b"0000:04:00.0", 60, numvfs=b"2\n"),
                                 fn(b"0000:04:00.4", 61, physfn=b"0000:04:00.0"),
                                 fn(b"0000:04:00.5", 62, physfn=b"0000:04:00.0")),
                            [NO_PF, 0, 0], [2, 0, 0], {60: 0, 61: 1, 62: 2}),
    "pf_on_vfio_without_vfs": (walk(fn(b"0000:04:00.0", 60, numvfs=b"0\n"),
                                    fn(b"0000:04:00.4", 61, physfn=b"0000:04:00.0")),
                               [NO_PF, 0], [0, 0], {60: VIABLE, 61: 1}),
    "physfn_uppercase": (walk(fn(b"0000:0a:00.0", 70), fn(b"0000:0a:00.4", 71, physfn=b"0000:0A:00.0")),
                         [NO_PF, NO_PF], [0, 0], {70: VIABLE, 71: VIABLE}),
    "physfn_missing": (walk(fn(b"0000:0a:00.0", 70), fn(b"0000:0a:00.4", 71)), [NO_PF, NO_PF], [0, 0],
                       {70: VIABLE, 71: VIABLE}),
    "physfn_read_failed": (walk(fn(b"0000:0a:00.0", 70), fn(b"0000:0a:00.4", 71, physfn=b"0000:0a:00.0", sflags=PHYSFN_ERR)),
                           [NO_PF, NO_PF], [0, 0], {70: VIABLE, 71: VIABLE}),
    "numvfs_read_failed": (walk(fn(b"0000:0a:00.0", 70, numvfs=b"3\n", sflags=NUMVFS_ERR)), [NO_PF], [0], {70: VIABLE}),
    "physfn_is_itself": (walk(fn(b"0000:0a:00.4", 71, physfn=b"0000:0a:00.4")), [NO_PF], [0], {71: VIABLE}),
    "pf_after_the_vf": (walk(fn(b"0000:0b:00.4", 81, physfn=b"0000:0b:00.0"), fn(b"0000:0b:00.0", 80)),
                        [1, NO_PF], [0, 0], {81: 0, 80: VIABLE}),
    "pf_not_in_the_walk": (walk(fn(b"0000:0c:00.4", 91, physfn=b"0000:0c:00.0")), [NO_PF], [0], {91: VIABLE}),
    "pf_unbound": (walk(fn(b"0000:0d:00.0", 100, driver=b"", flags=VC.DRIVER_ERR),
                        fn(b"0000:0d:00.4", 101, physfn=b"0000:0d:00.0")),
                   [NO_PF, 0], [0, 0], {101: VIABLE}),
    "pf_driver_read_failed": (walk(fn(b"0000:0d:00.0", 100, flags=VC.DRIVER_ERR),  # "vfio-pci" left in the field
                                   fn(b"0000:0d:00.4", 101, physfn=b"0000:0d:00.0")),
                              [NO_PF, 0], [0, 0], {101: VIABLE}),
    "pf_name_with_trailing_bytes": (walk(fn(b"0000:0e:00.0", 110), fn(b"0000:0e:00.4", 111, physfn=b"0000:0e:00.0x")),
                                    [NO_PF, NO_PF], [0, 0], {110: VIABLE, 111: VIABLE}),
    "duplicate_pf_names_first_wins": (walk(fn(b"0000:0f:00.0", 120, driver=b"nvidia"), fn(b"0000:0f:00.0", 121),
                                           fn(b"0000:0f:00.4", 122, physfn=b"0000:0f:00.0")),
                                      [NO_PF, NO_PF, 0], [0, 0, 0], {121: VIABLE, 122: VIABLE}),
    "mixed_groups": (walk(fn(b"0000:10:00.0", 130),                                   # a plain GPU
                          fn(b"0000:11:00.0", 131, numvfs=b"1\n"),                    # a PF with one VF
                          fn(b"0000:11:00.4", 130, physfn=b"0000:11:00.0"),           # its VF, in the GPU's group
                          fn(b"0000:12:00.0", 132, driver=b"nvidia"),                 # a PF on a host driver
                          fn(b"0000:12:00.4", 133, physfn=b"0000:12:00.0"),
                          fn(b"0000:12:00.5", 133, physfn=b"0000:12:00.0")),
                     [NO_PF, NO_PF, 1, NO_PF, 3, 3], [0, 1, 0, 0, 0, 0], {130: 2, 131: 1, 133: VIABLE}),
}
NUMVFS = [(b"0\n", 0), (b"7\n", 7), (b"07", 0), (b"", 0), (b"65536", 0), (b"65535\n", 65535), (b"-1", 0), (b"7", 7),
          (b"x\n", 0), (b"1\n\n", 0), (b"\n", 0), (b"1 \n", 0), (b"123456789", 0)]


@st.composite
def sriov_walks(draw):
    """Up to 40 records over 10 groups: PFs on vfio-pci, on a host driver or unbound, VFs naming one of them (or a PF
    outside the walk, itself, a malformed name), every sriov_numvfs shape of NUMVFS, and read-error flags."""
    n = draw(st.integers(0, 40))
    bdfs = [b"0000:%02x:00.%d" % (draw(st.integers(0, 5)), draw(st.integers(0, 7))) for _ in range(n)]
    rows = []
    for i in range(n):
        driver, flags = draw(st.sampled_from([(b"vfio-pci", 0), (b"vfio-pci", 0), (b"nvidia", 0), (b"", VC.DRIVER_ERR),
                                              (b"vfio-pci", VC.DRIVER_ERR)]))
        physfn = draw(st.sampled_from([b"", b"", b"0000:3f:00.0", b"0000:00:00.0", b"0000:00:20.0"] + bdfs))
        num = draw(st.sampled_from([b""] * 4 + [t for t, _ in NUMVFS]))
        sflags = draw(st.sampled_from([0] * 6 + [PHYSFN_ERR, NUMVFS_ERR]))
        rows.append((VC.rec(bdfs[i], draw(st.integers(0, 9)), driver=driver, flags=flags), sr(physfn, num, sflags)))
    return walk(*rows) if rows else (np.zeros(0, XO.DEVREC_DTYPE), np.zeros(0, SRIOVREC_DTYPE))


@st.composite
def forests(draw):
    """(recs, paths, group_off, group_members, pf_of): pyref_pcie-style walks where some records name another as PF;
    chains up to 8 keys, so a PF at depth 8 exercises the fallback."""
    n = draw(st.integers(0, 20))
    hb = ["pci0000:00", "pci0000:80"]
    mid = ["0000:00:01.0", "0000:00:02.0", "0000:01:00.0", "0000:02:00.0"]
    recs = np.zeros(n, XO.DEVREC_DTYPE)
    paths = np.zeros(n, PCIPATH_DTYPE)
    for i in range(n):
        bdf = "0000:%02x:00.%d" % (0x10 + i // 8, i % 8)
        comps = [draw(st.sampled_from(hb))] + draw(st.lists(st.sampled_from(mid), max_size=7)) + [bdf]
        text = "/".join(comps).encode()
        recs[i]["bdf"] = bdf.encode()
        paths[i]["path"] = text
        paths[i]["len"] = draw(st.sampled_from([len(text), len(text), 0]))
    pf_of = np.array([draw(st.sampled_from([NO_PF, NO_PF] + list(range(n)))) for _ in range(n)], np.uint32)
    order = draw(st.permutations(list(range(n))))
    keep = order[:draw(st.integers(0, n))]
    cuts = sorted(draw(st.lists(st.integers(0, len(keep)), max_size=6)))
    off = [0] + cuts + [len(keep)]
    return recs, paths, np.array(off, np.uint32), np.array(keep, np.uint32), pf_of



def deep(levels):
    """(recs, paths, group_off, group_members, pf_of): a PF whose chain has `levels` keys and its VF, one group each."""
    mids = ["0000:%02x:00.0" % (k + 1) for k in range(levels - 1)]
    recs = np.zeros(2, XO.DEVREC_DTYPE)
    paths = np.zeros(2, PCIPATH_DTYPE)
    for i, bdf in enumerate(["0000:40:00.0", "0000:40:00.1"]):
        text = "/".join(["pci0000:00"] + mids + [bdf]).encode()
        recs[i]["bdf"], paths[i]["path"], paths[i]["len"] = bdf.encode(), text, len(text)
    return recs, paths, np.array([0, 1, 2], np.uint32), np.array([0, 1], np.uint32), np.array([NO_PF, 0], np.uint32)
