"""Records for the tests of kxpu_pcie_tree_mdev: mdev record and path builders, the hand cases and a hypothesis strategy,
shared by the CPU and the GPU tests."""
import numpy as np
from hypothesis import strategies as st

from kxpu_b200.binding import MDEVREC_DTYPE, PCIPATH_DTYPE

MAX_DEPTH = 8
NO_NODE = 0xFFFFFFFF
# the worked example of the issue that introduced the call: a GPU at 0000:03:00.0 behind two switch levels
EXAMPLE_CHAIN = "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.0"


def uuid(k):
    """A canonical lowercase UUID numbered k."""
    h = "%032x" % (0x5d3b1c2e00004000a00000000000 + k)
    return "%s-%s-%s-%s-%s" % (h[:8], h[8:12], h[12:16], h[16:20], h[20:])


def rec(u, parent):
    r = np.zeros(1, MDEVREC_DTYPE)[0]
    r["uuid"] = u.encode()[:36] if len(u) == 36 else b""
    r["parent"] = parent.encode()
    return r


def path(text):
    """A kxpu_pcipath holding text, cut as the host does (over 120 bytes: unknown)."""
    p = np.zeros(1, PCIPATH_DTYPE)[0]
    b = text.encode()
    if 0 < len(b) <= 120:
        p["path"], p["len"] = b, len(b)
    return p


def mdev(u, parent, chain):
    """(record, path) of mdev u on parent function `parent` whose own path is `chain` (its link: chain/u)."""
    return rec(u, parent), path(chain + "/" + u)


def walk(rows, groups=None):
    """rows of (record, path) -> (recs, paths, group_off, group_members); groups: lists of record indices (default: one
    group per record)."""
    recs = np.array([r for r, _ in rows], MDEVREC_DTYPE)
    paths = np.array([p for _, p in rows], PCIPATH_DTYPE)
    groups = [[i] for i in range(len(rows))] if groups is None else groups
    off = np.zeros(len(groups) + 1, np.uint32)
    off[1:] = np.cumsum([len(g) for g in groups])
    mem = np.array([m for g in groups for m in g], np.uint32)
    return recs, paths, off, mem


def bridges(k):
    """A chain of k keys that ends in a function: k - 1 host bridges, then 0000:03:00.0 (the shortest text per key)."""
    return "/".join(["pci0000:%02x" % j for j in range(k - 1)] + ["0000:03:00.0"]), "0000:03:00.0"


def _deep(k):
    c, parent = bridges(k)
    return walk([mdev(uuid(k), parent, c)])


def _exact_len(total):
    """An mdev path of exactly `total` bytes (112..132): a host bridge and five functions, domains widened to 5..8 digits
    from the root down."""
    comps = ["pci0000:00", "0000:00:01.0", "0000:01:00.0", "0000:02:00.0", "0000:03:00.0", "0000:04:00.0"]
    extra = total - 112
    for j, c in enumerate(comps):
        x = min(4, extra)
        extra -= x
        if x:
            at = 3 if j == 0 else 0
            comps[j] = c[:at] + "1" + "0" * (3 + x) + c[at + 4:]
    assert extra == 0
    text = "/".join(comps)
    assert len(text) + 37 == total
    return walk([mdev(uuid(total), comps[-1], text)])


U0, U1, U2, U3 = uuid(0), uuid(1), uuid(2), uuid(3)
P_A, P_B = "0000:03:00.0", "0000:04:00.0"
SW = "pci0000:00/0000:00:01.0/0000:01:00.0"  # one switch with two down ports
HAND = {
    "example": walk([mdev(U0, P_A, EXAMPLE_CHAIN)]),
    "two_vgpus_one_gpu": walk([mdev(U0, P_A, EXAMPLE_CHAIN), mdev(U1, P_A, EXAMPLE_CHAIN)]),
    "two_gpus_one_switch": walk([mdev(U0, P_A, SW + "/0000:02:00.0/" + P_A), mdev(U1, P_B, SW + "/0000:02:01.0/" + P_B)]),
    "uuid_not_the_record": walk([(rec(U0, P_A), path(EXAMPLE_CHAIN + "/" + U1))]),
    "parent_not_the_record": walk([mdev(U0, P_B, EXAMPLE_CHAIN)]),
    "parent_a_host_bridge": walk([(rec(U0, "pci0000:00"), path("pci0000:00/" + U0))]),
    "uppercase_uuid": walk([(rec(U0.upper(), P_A), path(EXAMPLE_CHAIN + "/" + U0.upper()))]),
    "short_uuid": walk([(rec(U0[:35], P_A), path(EXAMPLE_CHAIN + "/" + U0[:35]))]),
    "uuid_without_dashes": walk([(rec(U0.replace("-", "") + "abcd", P_A), path(EXAMPLE_CHAIN + "/" + U0.replace("-", "") + "abcd"))]),
    "bdf_leaf": walk([(rec(U0, P_A), path(EXAMPLE_CHAIN))]),
    "len_119": _exact_len(119),
    "len_120": _exact_len(120),
    "len_121": _exact_len(121),
    "chain_of_1": walk([(rec(U0, P_A), path(P_A + "/" + U0))]),
    "chain_of_2": walk([mdev(U0, P_A, "pci0000:00/" + P_A)]),
    "chain_of_7": _deep(7),
    "chain_of_max_depth": _deep(MAX_DEPTH),
    "chain_of_max_depth_plus_1": _deep(MAX_DEPTH + 1),
    "vmd_domain": walk([mdev(U0, "10000:e1:00.0", "pci0000:00/0000:00:0e.0/pci10000:e0/10000:e0:06.0/10000:e1:00.0")]),
    "mdev_on_a_vf": walk([mdev(U0, "0000:03:00.4", SW + "/0000:02:00.0/0000:03:00.4"),
                          mdev(U1, "0000:03:00.5", SW + "/0000:02:00.0/0000:03:00.5")]),
    "group_unknown_and_known": walk([(rec(U0, P_A), path("")), mdev(U1, P_A, EXAMPLE_CHAIN)], groups=[[0, 1]]),
    "group_all_unknown": walk([(rec(U0, P_A), path("")), (rec(U1, P_A), path(EXAMPLE_CHAIN + "/" + U0))], groups=[[0, 1]]),
    "group_mixed_parents": walk([mdev(U0, P_A, SW + "/0000:02:00.0/" + P_A), mdev(U1, P_B, SW + "/0000:02:01.0/" + P_B),
                                 mdev(U2, P_A, SW + "/0000:02:00.0/" + P_A)], groups=[[0, 1], [2]]),
    "empty": walk([]),
}
# the chain length every hand case must get for its first record (0: unknown)
CHAIN_LEN = {
    "example": 5, "two_vgpus_one_gpu": 5, "two_gpus_one_switch": 5, "uuid_not_the_record": 0, "parent_not_the_record": 0,
    "parent_a_host_bridge": 0, "uppercase_uuid": 0, "short_uuid": 0, "uuid_without_dashes": 0, "bdf_leaf": 0,
    "len_119": 6, "len_120": 6, "len_121": 0, "chain_of_1": 0, "chain_of_2": 2, "chain_of_7": 7, "chain_of_max_depth": 0,
    "chain_of_max_depth_plus_1": 0, "vmd_domain": 5, "mdev_on_a_vf": 5, "group_unknown_and_known": 0,
    "group_all_unknown": 0, "group_mixed_parents": 5,
}


@st.composite
def mdev_walks(draw, max_n=24):
    """Walks over a small pool of functions, chains and UUIDs, so that groups share prefixes and parents, with the leaf
    and parent rules broken at random: a foreign or uppercase UUID, a foreign parent, a missing leaf, a cut or empty path,
    extra keys past the depth limit."""
    roots = ["pci0000:00", "pci0000:80", "pci10000:e0"]
    n = draw(st.integers(0, max_n))
    rows = []
    for i in range(n):
        dom = draw(st.sampled_from(roots))
        depth = draw(st.integers(0, 8))
        fns = ["%s:%02x:%02x.%d" % (dom[3:-3] if dom != "pci10000:e0" else "10000", draw(st.integers(0, 3)),
                                   draw(st.integers(0, 2)), draw(st.integers(0, 1))) for _ in range(depth)]
        comps = [dom] + fns
        parent = comps[-1] if fns else "0000:03:00.0"
        u = uuid(draw(st.integers(0, 5)))
        leaf = u
        fault = draw(st.sampled_from(["none"] * 6 + ["foreign_uuid", "upper", "foreign_parent", "no_leaf", "cut", "empty"]))
        if fault == "foreign_uuid":
            leaf = uuid(99)
        elif fault == "upper":
            leaf = u.upper()
        elif fault == "foreign_parent":
            parent = "0000:7f:00.0"
        text = "/".join(comps + ([] if fault == "no_leaf" else [leaf]))
        if fault == "cut":
            text = text[:draw(st.integers(1, len(text)))]
        r = rec(u, parent)
        rows.append((r, path("" if fault == "empty" else text)))
    order = draw(st.permutations(range(n)))
    groups, at = [], 0
    while at < n:
        k = draw(st.integers(1, 3))
        groups.append(list(order[at:at + k]))
        at += k
    return walk(rows, groups)
