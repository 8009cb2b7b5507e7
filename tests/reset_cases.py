"""Records for the reset tests (kxpu_reset_check): side-record builders, the reset_method texts, the hand-worked forests
and a hypothesis strategy, shared by the CPU and the GPU tests."""
import numpy as np
from hypothesis import strategies as st

import viab_cases as VC
from oracle import xpu_oracle as XO
from kxpu_b200.binding import PCIPATH_DTYPE, RESETREC_DTYPE

NV = VC.NV
VIABLE = 0xFFFFFFFF
SET_OK, NO_PATH, ROOT_BUS = 0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFFD
ABSENT, READ_ERR, LEGACY = 1, 2, 4
FLR, AF_FLR, PM, BUS, CXL_BUS, DEVICE_SPECIFIC, ACPI = 1, 2, 4, 8, 16, 32, 64
ALL, UNNAMED = 0x7F, 0x80


def rr(text=b"", flags=0):
    s = np.zeros(1, RESETREC_DTYPE)[0]
    s["txt"][:min(len(text), 64)] = np.frombuffer(text[:64], np.uint8)
    s["len"] = min(len(text), 65)
    s["flags"] = flags
    return s


def pp(comps, bdf):
    """the kxpu_pcipath of bdf below comps (host bridge first); comps None: unknown"""
    p = np.zeros(1, PCIPATH_DTYPE)[0]
    if comps is not None:
        text = "/".join(list(comps) + [bdf.decode()]).encode()
        p["path"], p["len"] = text, len(text)
    return p


def fn(bdf, group, comps, driver=b"vfio-pci", method=b"", rflags=ABSENT, flags=0, vendor=b"0x10de\n"):
    """(devrec, pcipath, resetrec) of one function: flags are the devrec's KXPU_REC_*, rflags the side record's."""
    return VC.rec(bdf, group, driver=driver, flags=flags, vendor=vendor), pp(comps, bdf), rr(method, rflags)


def walk(*rows):
    """rows of (devrec, pcipath, resetrec) -> (recs, paths, rrs)"""
    return (np.array([r for r, _, _ in rows], XO.DEVREC_DTYPE), np.array([p for _, p, _ in rows], PCIPATH_DTYPE),
            np.array([s for _, _, s in rows], RESETREC_DTYPE))


def m(text):
    """a present reset_method file holding text"""
    return dict(method=text, rflags=0)


ROOT = ["pci0000:40"]
PORT = ROOT + ["0000:40:01.0"]                                     # a root port
SWITCH = ["pci0000:00", "0000:00:01.0", "0000:01:00.0", "0000:02:08.0"]  # a switch's downstream port
VMD = ["pci0000:00", "0000:00:0e.0", "pci10000:e0"]                # a VMD domain below its endpoint

# name -> ((recs, paths, rrs), allow, methods, set_verdict, {group id: reset blocker or VIABLE}) under the NVIDIA class
HAND = {
    "flr_function": (walk(fn(b"0000:00:05.0", 10, ["pci0000:00"], **m(b"flr\n"))), ALL,
                     [FLR], [ROOT_BUS], {10: VIABLE}),
    "bus_only_alone_under_a_root_port": (walk(fn(b"0000:41:00.0", 11, PORT, **m(b"bus\n"))), ALL & ~BUS,
                                         [BUS], [SET_OK], {11: VIABLE}),
    "gpu_and_audio_one_group_under_a_switch_port": (
        walk(fn(b"0000:03:00.0", 20, SWITCH), fn(b"0000:03:00.1", 20, SWITCH)), ALL,
        [0, 0], [SET_OK, SET_OK], {20: VIABLE}),
    "audio_on_snd_hda_intel": (
        walk(fn(b"0000:03:00.0", 20, SWITCH), fn(b"0000:03:00.1", 20, SWITCH, driver=b"snd_hda_intel")), ALL,
        [0, 0], [1, 1], {20: 0}),
    "audio_in_another_group": (
        walk(fn(b"0000:03:00.0", 20, SWITCH), fn(b"0000:03:00.1", 21, SWITCH)), ALL,
        [0, 0], [1, 0], {20: 0, 21: 1}),
    "audio_in_another_group_with_flr": (
        walk(fn(b"0000:03:00.0", 20, SWITCH, **m(b"flr\n")), fn(b"0000:03:00.1", 21, SWITCH, **m(b"flr\n"))), ALL,
        [FLR, FLR], [1, 0], {20: VIABLE, 21: VIABLE}),
    "audio_unbound": (
        walk(fn(b"0000:03:00.0", 20, SWITCH), fn(b"0000:03:00.1", 20, SWITCH, driver=b"", flags=VC.DRIVER_ERR)), ALL,
        [0, 0], [1, 1], {20: 0}),
    "sibling_bridge_below_the_same_port": (
        walk(fn(b"0000:03:00.0", 30, SWITCH),
             fn(b"0000:03:01.0", 31, SWITCH, driver=b"pcieport", vendor=b"0x8086\n"),
             fn(b"0000:04:00.0", 30, SWITCH + ["0000:03:01.0"])), ALL,
        [0, 0, 0], [1, 1, SET_OK], {30: 0}),
    "three_groups_under_one_port": (
        walk(fn(b"0000:03:00.0", 42, SWITCH), fn(b"0000:03:00.1", 40, SWITCH), fn(b"0000:03:00.2", 41, SWITCH),
             fn(b"0000:03:00.3", 40, SWITCH)), ALL,
        [0, 0, 0, 0], [1, 0, 1, 0], {42: 0, 40: 1, 41: 2}),
    "root_bus": (walk(fn(b"0000:00:05.0", 50, ["pci0000:00"])), ALL, [0], [ROOT_BUS], {50: 0}),
    "vmd_domain_bus": (walk(fn(b"10000:e0:00.0", 51, VMD)), ALL, [0], [ROOT_BUS], {51: 0}),
    "vmd_below_a_port": (walk(fn(b"10000:e1:00.0", 52, VMD + ["10000:e0:01.0"])), ALL, [0], [SET_OK], {52: VIABLE}),
    "legacy_kernel_default": (walk(fn(b"0000:00:05.0", 60, ["pci0000:00"], rflags=ABSENT | LEGACY)), ALL,
                              [UNNAMED], [ROOT_BUS], {60: VIABLE}),
    "legacy_kernel_narrowed": (walk(fn(b"0000:00:05.0", 60, ["pci0000:00"], rflags=ABSENT | LEGACY)), FLR | PM,
                               [UNNAMED], [ROOT_BUS], {60: 0}),
    "method_outside_the_allow_list": (walk(fn(b"0000:00:05.0", 61, ["pci0000:00"], **m(b"pm\n"))), FLR,
                                      [PM], [ROOT_BUS], {61: 0}),
    "unknown_path": (walk(fn(b"0000:41:00.0", 62, None)), ALL, [0], [NO_PATH], {62: 0}),
    "unknown_path_with_flr": (walk(fn(b"0000:41:00.0", 62, None, **m(b"flr\n"))), ALL, [FLR], [NO_PATH], {62: VIABLE}),
    "read_error": (walk(fn(b"0000:00:05.0", 63, ["pci0000:00"], method=b"flr\n", rflags=READ_ERR)), ALL,
                   [0], [ROOT_BUS], {63: 0}),
    "second_member_blocks": (
        walk(fn(b"0000:00:05.0", 64, ["pci0000:00"], **m(b"flr\n")), fn(b"0000:00:05.1", 64, ["pci0000:00"])), ALL,
        [FLR, 0], [ROOT_BUS, ROOT_BUS], {64: 1}),
}

_T64 = (b"flr " * 16)[:63] + b"\n"
_T65 = (b"flr " * 17)[:64] + b"\n"
# (reset_method text, side-record flags, method bits)
TEXTS = [(name + b"\n", 0, 1 << k) for k, name in
         enumerate([b"flr", b"af_flr", b"pm", b"bus", b"cxl_bus", b"device_specific", b"acpi"])] + [
    (b"device_specific acpi flr af_flr pm bus cxl_bus\n", 0, ALL),
    (b"flr bus\n", 0, FLR | BUS), (b"flr flr\n", 0, FLR), (b"flr", 0, FLR), (b"", 0, 0), (b"\n", 0, 0),
    (b"FLR\n", 0, 0), (b"flrx\n", 0, 0), (b"fl\n", 0, 0), (b"warm flr\n", 0, FLR), (b"flr  bus\n", 0, FLR | BUS),
    (b" flr\n", 0, FLR), (b"flr \n", 0, FLR), (b"flr\n\n", 0, 0), (b"flr\nbus\n", 0, 0), (b"flr\tbus\n", 0, 0),
    (b"flr\0\n", 0, 0), (b"device_specifi\n", 0, 0), (b"device_specificx\n", 0, 0), (b"device_specific_x\n", 0, 0),
    (b"pm bus", 0, PM | BUS), (_T64, 0, FLR), (_T65, 0, 0), (b"x" * 200, 0, 0),
    (b"", ABSENT, 0), (b"", ABSENT | LEGACY, UNNAMED), (b"flr\n", ABSENT, 0), (b"flr\n", READ_ERR, 0),
    (b"flr\n", READ_ERR | ABSENT | LEGACY, 0), (b"bus\n", LEGACY, BUS),
]


def _child_bus(last):
    """(domain, bus) of a function directly below the path component last"""
    if last.startswith("pci"):
        dom, bus = last[3:].split(":")
        return dom, int(bus, 16)
    dom, bus, _ = last.split(":")
    return dom, int(bus, 16) + 1


@st.composite
def reset_walks(draw, max_n=40):
    """(recs, paths, rrs): up to max_n functions below a few host bridges, ports and switches (sibling bridges, root
    buses and VMD included), on vfio-pci, another class driver, a host driver or unbound, in a few groups, with every
    reset_method text of TEXTS and unknown paths."""
    n = draw(st.integers(0, max_n))
    parents = [["pci0000:00"], PORT, SWITCH, SWITCH + ["0000:03:01.0"], VMD, VMD + ["10000:e0:01.0"],
               ["pci0000:00", "0000:00:01.0"], ["pci0000:00", "0000:00:01.0", "0000:01:00.0"]]
    rows = []
    for _ in range(n):
        comps = draw(st.sampled_from(parents))
        dom, bus = _child_bus(comps[-1])
        bdf = ("%s:%02x:%02x.%d" % (dom, bus, draw(st.integers(0, 2)), draw(st.integers(0, 7)))).encode()
        if draw(st.integers(0, 9)) == 0:
            comps = None
        driver, flags = draw(st.sampled_from([(b"vfio-pci", 0)] * 4 + [(b"pcieport", 0), (b"nvme", 0),
                                              (b"", VC.DRIVER_ERR), (b"vfio-pci", VC.IOMMU_ERR)]))
        text, rflags, _ = draw(st.sampled_from(TEXTS))
        rows.append(fn(bdf, draw(st.integers(0, 4)), comps, driver=driver, flags=flags, method=text, rflags=rflags))
    if not rows:
        return np.zeros(0, XO.DEVREC_DTYPE), np.zeros(0, PCIPATH_DTYPE), np.zeros(0, RESETREC_DTYPE)
    return walk(*rows)


ALLOWS = [ALL, 0, FLR, FLR | PM, BUS, ALL & ~BUS]
