"""GetPreferredAllocation at its edges (include/kxpu.h: kxpu_preferred_allocation, kxpu_preferred_allocation_pcie):
hand-built forests whose answers are worked out by hand from the rule, the null-device padding that sends any request
through the large shape, and generators for the large shape's tile seams, CTA strides and back-to-back requests.

The node key of the PCIe call is (avail, -depth, the ancestors' avail from the parent up, lowest available position).
Each hand case below isolates one term of it, or one step of the NUMA bin order, and is built so that a rule that
skips or reverses that term picks a different answer (most often: the winner holds the higher positions and the higher
node ids, so a tie broken by position or node id alone goes the other way).
"""
import numpy as np

NO = 0xFFFFFFFF
MAX_DEPTH = 8
TILE = 4096      # topology.cu k_big_scatter: device positions per tile
WARP_MAX = 256   # topology.cu: larger requests take the large shape


class Case:
    """A device list (dev_numa, dev_node) over a forest (parent, depth), requests [(available, must, size)] and the
    answer worked out by hand for each.  numa: no device is in a node, so both calls give the same answer."""

    def __init__(self, name, dev_numa, dev_node, parent, requests, answers):
        self.name = name
        self.dev_numa = np.array(dev_numa, np.uint64)
        self.dev_node = np.array(dev_node, np.uint32)
        self.parent = np.array(parent, np.uint32)
        self.depth = depths(parent)
        self.requests, self.answers = requests, answers
        self.numa = bool((self.dev_node == NO).all())

    def __repr__(self):
        return self.name


def depths(parent):
    d = []
    for p in parent:
        d.append(0 if p == NO else d[p] + 1)
    return np.array(d, np.uint8)


def chains(specs):
    """One chain of nodes per spec, root first; spec[t] = the devices placed directly in the chain's node at depth t,
    and the leaf (depth len(spec)) holds two devices.  Chains are laid out one after the other, so a later chain holds
    higher positions and higher node ids.  Returns (dev_node, parent, leaves): leaves[i] = chain i's leaf devices."""
    dev_node, parent, leaves = [], [], []
    for spec in specs:
        base = len(parent)
        for t in range(len(spec) + 1):
            parent.append(NO if t == 0 else base + t - 1)
        for t, k in enumerate(spec):
            dev_node += [base + t] * k
        leaves.append([len(dev_node), len(dev_node) + 1])
        dev_node += [base + len(spec)] * 2
    return dev_node, parent, leaves


def _chain_case(name, specs, winner):
    dev_node, parent, leaves = chains(specs)
    n = len(dev_node)
    avail = list(range(n))[::-1]  # descending: the answer may not depend on the list order
    c = Case(name, [1] * n, dev_node, parent, [(avail, [], 2)], [leaves[winner]])
    c.leaves = leaves
    return c


def _hand():
    cases = []
    # avail ties (2) between a depth-1 leaf whose root also holds only those two devices and a depth-2 leaf: the
    # deeper leaf wins; a rule that prefers the shallower node takes the first chain's root
    cases.append(_chain_case("depth_decides", [[0], [1, 1]], 1))
    # equal avail and depth; the parents' avail (4 vs 3) decides for the second chain while the roots' (7 vs 8) point
    # the other way, so walking the ancestors root first picks the first chain
    cases.append(_chain_case("parent_decides", [[3, 2], [5, 1]], 1))
    # equal through the parents (3, 3); the grandparents' (5 vs 4) decide, the roots' (5 vs 8) point the other way
    cases.append(_chain_case("grandparent_decides", [[0, 2, 1], [4, 1, 1]], 1))
    # leaves at depth 7 (KXPU_PCIE_MAX_DEPTH - 1), every ancestor equal but the roots (4 vs 3)
    cases.append(_chain_case("depth7_root_decides", [[2] + [0] * 6, [1] + [0] * 6], 1))
    # siblings equal in avail, depth and parent: the lowest available position decides, and it sits in the
    # higher node id
    cases.append(Case("siblings_lowest_position", [1] * 4, [2, 2, 1, 1], [NO, 0, 0], [([3, 1, 2, 0], [], 2)],
                      [[0, 1]]))
    # an exact fit (avail 3 = size) against a deeper node of 4 and its parent of 5, all under one root
    cases.append(Case("exact_fit", [1] * 8, [3, 3, 3, 3, 2, 1, 1, 1], [NO, 0, 0, 2], [(list(range(8)), [], 3)],
                      [[5, 6, 7]]))
    # the must-include device 3 keeps node 1 (2 devices, the best fit without it) from qualifying: X = node 2
    cases.append(Case("must_decides", [1] * 5, [1, 1, 2, 2, 2], [NO, 0, 0], [([4, 3, 2, 1, 0], [3], 2)], [[3, 2]]))
    # the must-include device 4 is in no node, so no node qualifies and X is every device; U = {1} puts home 1 first
    cases.append(Case("must_in_no_node", [1, 1, 2, 2, 2], [1, 1, 1, 1, NO], [NO, 0], [([0, 1, 2, 3, 4], [4], 3)],
                      [[4, 2, 3]]))
    # lca levels: a chain of nodes 0..7 (node t at depth t), the must-include device 8 in node 7 and one candidate in
    # each node t at position t, so the candidate of depth t has lca depth t; device 9 in another root and device 10 in
    # no node have none.  Homes alternate 0 / 1 with the depth, U = {1}: without the levels home 1 would come first.
    # X is every device (the chain holds 9 of 11).
    numa = [1 << (t % 2) for t in range(8)] + [2, 1, 2]
    node = list(range(8)) + [7, 8, NO]
    full = [8, 7, 6, 5, 4, 3, 2, 1, 0, 10, 9]
    avail = [3, 9, 0, 10, 7, 1, 8, 5, 2, 6, 4]
    cases.append(Case("lca_levels", numa, node, [NO] + list(range(7)) + [NO],
                      [(avail, [8], 11), (avail, [8], 4), (avail, [8], 1)], [full, full[:4], [8]]))
    # NUMA bins, no device in a node: homes 0 (mask 1 and the all-ones mask), 1 (a two-node mask too), 62, 63 (bit 63
    # only) and 64 (mask 0)
    homes = [1 << 63, (1 << 64) - 1, 1 << 62, 0, 2, 1 << 63, 0, 1, 1 << 62, 2 | 32, 1 << 63, 2, 2]
    #        63       0              62       64 1  63       64 0  62       1       63       1  1
    n = len(homes)
    shuffled = [3, 10, 7, 0, 12, 8, 1, 5, 2, 11, 9, 4, 6]
    cases.append(Case("numa_bins", homes, [NO] * n, [], [
        # U empty: c = {1: 4, 63: 3, 0: 2, 62: 2} -- the tie of 0 and 62 goes to the lower k -- then 64
        (list(range(n))[::-1], [], n),
        # must [10, 1] (descending, kept in request order): U = {63, 0}; group 0: 63 (2 left) before 0 (1 left),
        # ahead of group 1: 1 (4) and 62 (2), then 64
        (shuffled, [10, 1], n),
        (shuffled, [10, 1], 5),
        # a must-include device of home 64 adds nothing to U
        (list(range(n)), [3], 3),
    ], [
        [4, 9, 11, 12, 0, 5, 10, 1, 7, 2, 8, 3, 6],
        [10, 1, 0, 5, 7, 4, 9, 11, 12, 2, 8, 3, 6],
        [10, 1, 0, 5, 7],
        [3, 4, 9],
    ]))
    return {c.name: c for c in cases}


HAND = _hand()


def pad(dev_numa, dev_node, requests, n_pad, seed=0):
    """Null devices: n_pad positions after every real device, NUMA mask 0 and no node, mixed into every request's
    available list.  They change no node count and add candidates only to bin 64 at the lowest level, where they sort
    after every original candidate, so each request keeps its answer.  With n_pad >= 257 every request takes the large
    shape."""
    rng = np.random.default_rng(seed)
    n = len(dev_numa)
    numa = np.concatenate([np.asarray(dev_numa, np.uint64), np.zeros(n_pad, np.uint64)])
    node = None if dev_node is None else np.concatenate([np.asarray(dev_node, np.uint32), np.full(n_pad, NO, np.uint32)])
    out = []
    for av, mu, size in requests:
        av = np.concatenate([np.asarray(av, np.int64), np.arange(n, n + n_pad)])
        out.append((av[rng.permutation(len(av))].astype(np.uint32), np.asarray(mu, np.uint32), size))
    return numa, node, out


# ---------------------------------------------------------------- the large shape
def range_forest(n_devs, spans=(8192, 2048, 512, 64), none_every=97):
    """A forest over device positions in walk order: a node at depth t for every spans[t] positions, each inside its
    parent's range (so deep lca levels lie in one tile and shallow ones span tiles); every none_every-th device is in
    no node.  Node ids are assigned root first, in position order.  Returns (dev_node, parent, depth)."""
    parent, dev_node = [], np.full(n_devs, NO, np.uint32)

    def build(lo, hi, t, par):
        v = len(parent)
        parent.append(par)
        if t + 1 == len(spans):
            dev_node[lo:hi] = v
            return
        for a in range(lo, hi, spans[t + 1]):
            build(a, min(a + spans[t + 1], hi), t + 1, v)

    for a in range(0, n_devs, spans[0]):
        build(a, min(a + spans[0], n_devs), 0, NO)
    dev_node[::none_every] = NO
    parent = np.array(parent, np.uint32)
    return dev_node, parent, depths(parent)


def range_numa(n_devs, nodes=4, seed=5):
    """Homes by position range, 5 % unknown, 2 % on two nodes (so the bins cut across the tiles)."""
    rng = np.random.default_rng(seed)
    k = np.arange(n_devs, dtype=np.int64) * nodes // max(n_devs, 1)
    m = np.uint64(1) << k.astype(np.uint64)
    m = np.where(rng.random(n_devs) < 0.02, m | (np.uint64(1) << ((k + 1) % nodes).astype(np.uint64)), m)
    return np.where(rng.random(n_devs) < 0.05, np.uint64(0), m).astype(np.uint64)


def seam_must(n_devs, dev_node):
    """Two must-include devices: one in the deepest node at the end (its deep lca levels then lie in the last tile
    only, behind empty tiles; in front of it when the last tile holds one position, which must stay a candidate) and
    one in no node (so no node qualifies and X is every device, whatever the size)."""
    deep = n_devs - 2 if (n_devs - 1) % TILE == 0 or dev_node[n_devs - 1] == NO else n_devs - 1
    none = int(np.flatnonzero(dev_node == NO)[0])
    return [deep, none]


def seam_sizes(order, nm, most=4):
    """Sizes whose r = size - nm ends on the last candidate in front of a tile seam and on the first behind it, given
    the full candidate order of a request (its answer with size = |available|).  A seam is a step to a higher tile
    between neighbours in that order (the same bin: positions ascend inside a bin)."""
    c = order[nm:]
    seams = [i for i in range(1, len(c)) if c[i - 1] // TILE < c[i] // TILE]
    assert seams, "no tile seam in the candidate order"
    pick = sorted({seams[0], seams[len(seams) // 2], seams[-1]} | set(seams[:most - 3]))
    sizes = []
    for i in pick:
        assert c[i - 1] // TILE < c[i] // TILE
        sizes += [nm + i, nm + i + 1]
    return sizes
