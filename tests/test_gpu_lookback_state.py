"""GPU tests of the look-back state over a context's life, against the oracles.

Every output whose size depends on the data comes out of a decoupled look-back over one per-context buffer of tile
status words (csrc/scan.cuh).  A word carries the 24-bit epoch of the call that wrote it, and a word whose epoch is not
the running call's counts as not yet published.  So no word may carry the running call's epoch unless this call wrote
it: the buffer is zeroed on the context's stream when it is allocated or grown, and again whenever the epoch wraps.
KXPU_SCAN_EPOCH_LIMIT moves the wrap from 2^24 down to a few epochs, so that a test can run it hundreds of times over
buffers full of words of earlier calls.

The look-back users and their tiles (a call of one tile never reads a predecessor's word, so every call here spans at
least two; the Call objects below restate the host code's sizes and every test asserts it):

  scan_kernel    names, alloc_names(_kind), mdev_names, lw_encode(_topo)   4096 items (n + 1 are scanned)  1 epoch
  k_cdi_fused    cdi_emit(_kind, _mdev)                                    128 devices                     1 epoch
  k_cdi_decode   cdi_parse(_mdev, _cdev, _mdev_cdev, _vf_vgpu[_cdev])      8192 bytes                      1 epoch
                 (tests/test_gpu_cdi_edges.py interleaves it with the emits of all six layouts under the epoch wrap)
  classify       classify(_rules, _mdev, _topo, _mdev_topo)                2048 / 4096 records   3 + 1 per sort pass,
                                                                                                 twice on the retry
  k_rc_probe     reconcile                                                 1024 entries                    1 epoch
  k_big_scatter  preferred_allocation                                      4096 device positions  1 per request of
                                                                                                  > 256 positions
"""
import threading

import numpy as np
import pytest

from oracle import mdev_oracle as MO
from oracle import reconcile_oracle as RO
from oracle import topo_oracle as TO
from oracle import xpu_oracle as XO

pytestmark = pytest.mark.gpu

SCAN_TILE = 4096               # scan.cuh SCAN_TILE
EMIT_TILE = 128                # emit.cu TILE
C_TILE, OS_TILE = 2048, 4096   # classify.cu: the accept / device-first scans, the one-sweep sort
RC_TILE = 1024                 # reconcile.cu RC_TILE
BS_TILE, BINS = 4096, 65       # topology.cu k_big_scatter: positions per tile, status words per tile
WARP_MAX = 256                 # topology.cu: larger requests take k_big_scatter
FIRST_WORDS = 1 << 14          # kx_scan_state: the first buffer of a context
KIND = b"amd.com/gpu"
MDEV_KIND = b"nvidia.com/vgpu"
NV = [(b"10de", b"vfio-pci")]


def cdiv(a, b):
    return (a + b - 1) // b


def sort_passes(n):
    """classify_once: 8-bit radix passes over keys of bits_for(n) bits."""
    b = 1
    while b < 32 and (1 << b) < n + 1:
        b += 1
    return (b + 7) // 8


class Call:
    """One look-back call: op and inputs, the oracle's answer, and what it asks of the state: the epochs it takes,
    the status words it needs and the tiles of its shortest look-back."""

    def __init__(self, op, args, want, epochs, words, tiles):
        self.op, self.args, self.want = op, args, want
        self.epochs, self.words, self.tiles = epochs, words, tiles

    def __repr__(self):
        return "%s(tiles=%d, words=%d, epochs=%d)" % (self.op, self.tiles, self.words, self.epochs)


def scan_call(op, args, want, n, calls=1):
    """calls = 2: the binding sizes the output with a first call (out = NULL), which runs the look-back too."""
    return Call(op, args, want, calls, cdiv(n + 1, SCAN_TILE), cdiv(n + 1, SCAN_TILE))


def classify_call(op, args, want, n, retry=False):
    # three scans over C_TILE tiles + the two sorts' per-digit words over OS_TILE tiles (classify_once's st_words)
    words = 3 * cdiv(n, C_TILE) + 2 * cdiv(n, OS_TILE) * 256
    return Call(op, args, want, (3 + sort_passes(n)) * (2 if retry else 1), words, min(cdiv(n, C_TILE), cdiv(n, OS_TILE)))


class Cases:
    """Inputs and oracle answers, built once per module.  Every builder takes a seed, so a sequence is a script."""

    def __init__(self, oracle, workloads, text, orows):
        self.O, self.W, self.text, self.orows = oracle, workloads, text, orows
        self.keys = orows["key"]
        self.mdev_pool = workloads.mdev_records(1 << 14, seed=21)

    def classify(self, n, seed):
        recs = self.W.cfg3_records(self.keys, n, seed)
        return classify_call("classify", (recs,), self.O.classify(recs), n)

    def classify_rules(self, n, seed):
        recs = self.W.xpu_records(self.keys, n, seed)
        return classify_call("classify_rules", (self.W.XPU_RULES, recs), XO.classify_rules(self.W.XPU_RULES, recs), n)

    def classify_mdev(self, n, seed):
        n = cdiv(n, 16) * 16  # mdev_records: 16 mdevs per parent
        recs = self.W.mdev_records(n, seed)
        return classify_call("classify_mdev", (self.W.MDEV_RULES, recs), MO.classify_mdev(self.W.MDEV_RULES, recs), n)

    def classify_topo(self, n, seed):
        recs = self.W.topo_records(self.keys, n, 4, seed)
        return classify_call("classify_topo", (NV, recs, False), TO.classify_topo(NV, recs), n)

    def classify_mdev_topo(self, n, seed):
        n = cdiv(n, 16) * 16
        recs = self.W.topo_mdev_records(n, 4, seed)
        rules = self.W.MDEV_RULES
        return classify_call("classify_topo", (rules, recs, True), TO.classify_topo(rules, recs, mdev=True), n)

    def classify_retry(self, n=200000):
        """Distinct 5-digit device ids, each record its own group: more ids than the 2^17 slots of the first device-id
        table, so classify runs a second time with a full-size table (test_classify_sizes_and_degenerate's input)."""
        recs = np.zeros(n, dtype=self.O.DEVREC_DTYPE)
        recs["bdf"] = self.W.enumerate_bdfs(n).view("S16").reshape(n)
        recs["vendor_txt"] = np.frombuffer(b"0x10de\n\0", np.uint8)
        recs["device_txt"] = np.frombuffer(b"".join(b"0x%05x\n" % i for i in range(n)), np.uint8).reshape(n, 8)
        recs["vendor_len"], recs["device_len"] = 7, 8
        recs["driver"] = b"vfio-pci"
        recs["iommu_group"] = np.arange(n, dtype=np.uint32)
        want = self.O.classify(recs)
        assert want["n_devids"] == n > (1 << 17)
        return classify_call("classify", (recs,), want, n, retry=True)

    def names(self, n, seed):
        sel = np.random.default_rng(seed).integers(0, len(self.orows), n)
        return scan_call("names", (sel,), self.O.names_bulk(self.text, self.orows["line_off"][sel]), n, 2)

    def alloc_names(self, n, seed, kind=None):
        idx = np.random.default_rng(seed).integers(0, 1 << 40, n, dtype=np.uint64)
        idx >>= np.random.default_rng(seed + 1).integers(0, 40, n).astype(np.uint64)  # every digit count
        if kind is None:
            return scan_call("alloc_names", (idx, None), self.O.alloc_names(idx), n)
        return scan_call("alloc_names", (idx, kind), XO.alloc_names_kind(kind, idx), n)

    def mdev_names(self, n, seed):
        idx = np.random.default_rng(seed).integers(0, len(self.mdev_pool), n).astype(np.uint32)
        return scan_call("mdev_names", (self.mdev_pool, idx), MO.mdev_names(self.mdev_pool, idx), n, 2)

    def lw_encode(self, n, seed, topo=False):
        rng = np.random.default_rng(seed)
        g = rng.integers(0, 2**32 - 1, n, dtype=np.uint64).astype(np.uint32)
        h = (rng.random(n) < 0.8).astype(np.uint8)
        if not topo:
            return scan_call("lw_encode", (g, h), self.O.lw_encode(g, h), n, 2)
        m = np.where(rng.random(n) < 0.3, 0, np.uint64(1) << rng.integers(0, 64, n).astype(np.uint64)).astype(np.uint64)
        return scan_call("lw_encode_topo", (g, h, m), TO.lw_encode_topo(g, h, m), n, 2)

    def cdi_emit(self, n, seed, kind=None):
        rng = np.random.default_rng(seed)
        devs = self.W.cfg5_devices(n)
        devs["index"] = rng.integers(0, 2**63, n, dtype=np.uint64) >> rng.integers(0, 63, n).astype(np.uint64)
        devs["iommu_group"] = rng.integers(0, 2**32 - 1, n, dtype=np.uint64).astype(np.uint32)
        fmt = int(rng.integers(0, 2))
        want = self.O.cdi_emit(fmt, devs) if kind is None else XO.cdi_emit_kind(fmt, kind, devs)
        return Call("cdi_emit", (fmt, devs, kind), want, 1, cdiv(n, EMIT_TILE), cdiv(n, EMIT_TILE))

    def cdi_emit_mdev(self, n, seed):
        devs = self.W.mdev_devices(n, seed)
        fmt = seed & 1
        return Call("cdi_emit_mdev", (fmt, devs, MDEV_KIND), MO.cdi_emit_mdev(fmt, MDEV_KIND, devs), 2, cdiv(n, EMIT_TILE),
                    cdiv(n, EMIT_TILE))

    def reconcile(self, n, seed):
        prev, cur, ni = self.W.reconcile_pair(seed, n, mdev=bool(seed & 1))
        t = cdiv(len(cur), RC_TILE)
        return Call("reconcile", (prev, cur, ni), RO.reconcile(prev, cur, ni), 1, t, t)

    def preferred_allocation(self, k, n_big, n_warp, seed):
        """n_devs = 4096 k + 1: k full tiles and a last tile of one position.  n_big requests of more than 256
        positions (one over every device) and n_warp of at most 256, interleaved."""
        rng = np.random.default_rng(seed)
        n_devs = BS_TILE * k + 1
        dev_numa = self.W.topo_dev_numa(n_devs, nodes=4, seed=seed)
        reqs = []
        sizes = [n_devs] + [int(rng.integers(WARP_MAX + 1, n_devs + 1)) for _ in range(n_big - 1)]
        sizes += [int(rng.integers(0, WARP_MAX + 1)) for _ in range(n_warp)]
        for na in rng.permutation(np.array(sizes[:n_big + n_warp], np.int64)).tolist():
            av = rng.permutation(n_devs)[:na].astype(np.uint32)
            mu = av[rng.permutation(na)[:int(rng.integers(0, min(na, 3) + 1))]]
            reqs.append((av, mu, int(rng.integers(len(mu), na + 1))))
        nb = sum(len(r[0]) > WARP_MAX for r in reqs)
        assert nb == n_big
        t = cdiv(n_devs, BS_TILE)
        return Call("preferred_allocation", (dev_numa, reqs), TO.preferred_allocation(dev_numa, reqs), nb, t * BINS, t)


def same(got, want, what):
    if isinstance(want, dict):
        assert set(want) <= set(got), what
        for k in want:
            same(got[k], want[k], "%s.%s" % (what, k))
    elif isinstance(want, tuple):
        assert len(got) == len(want), what
        for i, (g, w) in enumerate(zip(got, want)):
            same(g, w, "%s[%d]" % (what, i))
    elif isinstance(want, np.ndarray):
        assert np.array_equal(np.asarray(got), want), what
    else:
        assert got == want, what


def load_names_table(kx, text, orows):
    """pci.ids on kx (no look-back: the parse keeps its own words); returns the table and its rows in oracle order."""
    tab = kx.pciids_load(text)
    keys, offs, rows = kx.table_export(tab)
    assert np.array_equal(keys, orows["key"]) and np.array_equal(offs, orows["line_off"])
    return tab, rows


def run(kx, c, what, tab=None, rows=None):
    a = c.args
    if c.op == "classify":
        got = kx.classify(a[0])
    elif c.op == "classify_rules":
        got = kx.classify_rules(a[0], a[1])
    elif c.op == "classify_mdev":
        got = kx.classify_mdev(a[0], a[1])
    elif c.op == "classify_topo":
        got = kx.classify_topo(a[0], a[1], mdev=a[2])
    elif c.op == "names":
        got = kx.names_blob(tab, rows[a[0]])
    elif c.op == "alloc_names":
        got = kx.alloc_names(a[0], a[1])
    elif c.op == "mdev_names":
        got = kx.mdev_names(a[0], a[1])
    elif c.op == "lw_encode":
        got = kx.lw_encode(a[0], a[1])
    elif c.op == "lw_encode_topo":
        got = kx.lw_encode_topo(a[0], a[1], a[2])
    elif c.op == "cdi_emit":
        got = kx.cdi_emit(a[0], a[1], a[2])
    elif c.op == "cdi_emit_mdev":
        got = kx.cdi_emit_mdev(a[0], a[1], a[2])
    elif c.op == "reconcile":
        got = kx.reconcile(a[0], a[1], a[2])
    elif c.op == "preferred_allocation":
        got = kx.preferred_allocation(a[0], a[1])
    else:
        raise AssertionError(c.op)
    same(got, c.want, "%s %r" % (what, c))


@pytest.fixture
def fresh(monkeypatch):
    """fresh(**env) -> a new context created under the given KXPU_* environment; closed at teardown (a context the
    test closed itself is skipped)."""
    import kxpu_b200 as K
    made = []

    def make(**env):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        k = K.Kxpu(0)
        made.append(k)
        return k
    yield make
    for k in made:
        k.close()


@pytest.fixture(scope="module")
def cases(oracle, workloads, pci_text, oracle_rows):
    return Cases(oracle, workloads, pci_text, oracle_rows)


def small_round(cs, seed):
    """One multi-tile call of every look-back user (every entry point of the table above), within the first buffer."""
    return [cs.classify(4097 + 37 * seed, seed), cs.names(4096 + 101 * seed, seed), cs.alloc_names(4096 + 59 * seed, seed),
            cs.cdi_emit(129 + 41 * seed, seed), cs.reconcile(1100 + 7 * seed, seed),
            cs.alloc_names(5000 + 13 * seed, seed, KIND), cs.classify_rules(6000 + 11 * seed, seed),
            cs.cdi_emit(300 + 5 * seed, seed, KIND), cs.mdev_names(4100 + 3 * seed, seed),
            cs.classify_mdev(4500 + 17 * seed, seed), cs.cdi_emit_mdev(257 + 9 * seed, seed),
            cs.lw_encode(4200 + 23 * seed, seed), cs.lw_encode(4096 + 29 * seed, seed, topo=True),
            cs.classify_topo(5000 + 31 * seed, seed), cs.classify_mdev_topo(4200 + 19 * seed, seed),
            cs.preferred_allocation(1 + seed % 2, 3, 5, seed)]


@pytest.fixture(scope="module")
def life_script(cases):
    return daemon_script(cases)


def daemon_script(cases):
    """The daemon's life: a start-up round that fits the first 2^14-word buffer, a 2^18-record classify that grows it,
    then a seeded mix of smaller calls (so words of the large call lie beyond their tiles) with the device-id retry and
    preferred allocations of many large requests in it."""
    first = small_round(cases, 0)
    grow = [cases.classify(1 << 18, 100)]
    rest = small_round(cases, 1) + small_round(cases, 2) + [
        cases.classify_retry(), cases.preferred_allocation(2, 12, 20, 101), cases.preferred_allocation(3, 10, 4, 102),
        cases.preferred_allocation(1, 16, 0, 103), cases.classify_topo(70000, 104), cases.reconcile(5000, 105),
        cases.names(20000, 106), cases.cdi_emit(3000, 107)]
    order = np.random.default_rng(2024).permutation(len(rest))
    script = first + grow + [rest[i] for i in order] + small_round(cases, 3)
    assert all(c.words <= FIRST_WORDS for c in first)
    assert grow[0].words > FIRST_WORDS and sort_passes(1 << 18) == 3 and grow[0].words == 33152
    assert all(c.words < grow[0].words for c in script[len(first) + 1:])
    return script


def check_multi_tile(calls):
    bad = [c for c in calls if c.tiles < 2]
    assert not bad, bad


@pytest.mark.parametrize("limit", ["2", "3", "5", "64", None, "0", "1", "16777217", "abc"],
                         ids=["limit2", "limit3", "limit5", "limit64", "default", "bad0", "bad1", "bad16777217", "badabc"])
def test_daemon_life_across_wraps(limit, fresh, monkeypatch, life_script, pci_text, oracle_rows):
    """One long-lived context runs the daemon's scripted life of 73 calls (every entry point that uses the state; 238
    epochs, counting the binding's sizing calls and the classify retry) under KXPU_SCAN_EPOCH_LIMIT = limit.  With
    limit 64 every epoch value 1..63 is taken at least three times, over words that earlier calls left with the same
    value; with 2 .. 5 the wrap also falls inside single calls (the classify epochs, the large requests of one
    preferred allocation).  The values 0, 1, 2^24 + 1 and "abc" are not
    accepted and leave the default 2^24.  Fails when the wrap's zeroing is missing or not ordered in front of the next
    look-back on the stream: a stale word carrying the running epoch is read as a predecessor's prefix, and a size,
    an offset or a sort position comes out wrong."""
    script = life_script
    check_multi_tile(script)
    epochs = sum(c.epochs for c in script)
    assert len(script) == 73 and epochs == 238 >= 3 * 63  # limit 64: each of the 63 values taken at least three times
    if limit is None:
        monkeypatch.delenv("KXPU_SCAN_EPOCH_LIMIT", raising=False)
        kx = fresh()
    else:
        kx = fresh(KXPU_SCAN_EPOCH_LIMIT=limit)
    tab, rows = load_names_table(kx, pci_text, oracle_rows)
    try:
        for i, c in enumerate(script):
            run(kx, c, "call %d" % i, tab, rows)
    finally:
        tab.free()


ENTRY_POINTS = ["names", "alloc_names", "alloc_names_kind", "mdev_names", "lw_encode", "lw_encode_topo", "cdi_emit",
                "cdi_emit_kind", "cdi_emit_mdev", "classify", "classify_rules", "classify_mdev", "classify_topo",
                "classify_mdev_topo", "reconcile", "preferred_allocation"]


@pytest.fixture(scope="module")
def first_calls(cases):
    """Per entry point, a multi-tile first call (inputs unlike the history's)."""
    s = 50
    return dict(names=cases.names(9000, s), alloc_names=cases.alloc_names(9000, s), alloc_names_kind=cases.alloc_names(7000, s, KIND),
                mdev_names=cases.mdev_names(8000, s), lw_encode=cases.lw_encode(8192, s),
                lw_encode_topo=cases.lw_encode(6000, s, topo=True), cdi_emit=cases.cdi_emit(1000, s),
                cdi_emit_kind=cases.cdi_emit(700, s, KIND), cdi_emit_mdev=cases.cdi_emit_mdev(900, s),
                classify=cases.classify(9000, s), classify_rules=cases.classify_rules(9000, s),
                classify_mdev=cases.classify_mdev(9000, s), classify_topo=cases.classify_topo(9000, s),
                classify_mdev_topo=cases.classify_mdev_topo(9000, s), reconcile=cases.reconcile(4000, s),
                preferred_allocation=cases.preferred_allocation(2, 4, 4, s))


@pytest.mark.parametrize("entry", ENTRY_POINTS)
def test_first_lookback_call_of_a_fresh_context(entry, fresh, monkeypatch, life_script, first_calls, pci_text, oracle_rows):
    """A context runs 20 multi-tile calls and is destroyed; then a new context makes `entry`'s first look-back call.
    Both buffers are the first 2^14 words, so the new one can be the old one's memory, holding words with epochs
    1, 2, 3 ..., the very epochs the new context's first calls use.  Fails when the new buffer's zeroing is not ordered
    in front of that first look-back (the context's stream does not wait for the legacy stream)."""
    monkeypatch.delenv("KXPU_SCAN_EPOCH_LIMIT", raising=False)
    history = [c for c in life_script[:16] + life_script[-16:] if c.op != "names"][:20]
    first = first_calls[entry]
    check_multi_tile(history + [first])
    assert all(c.words <= FIRST_WORDS for c in history + [first])
    old = fresh()
    for i, c in enumerate(history):
        run(old, c, "old context, call %d" % i)
    old.close()
    kx = fresh()
    tab = rows = None
    if entry == "names":
        tab, rows = load_names_table(kx, pci_text, oracle_rows)
    try:
        run(kx, first, "first call", tab, rows)
    finally:
        if tab is not None:
            tab.free()


def test_mixed_callers_on_one_context(fresh, cases, pci_text, oracle_rows):
    """8 threads share one context with KXPU_SCAN_EPOCH_LIMIT=5, so the epoch wraps every few calls while other
    threads wait on the context's lock.  Four rediscovery-shaped threads run classify_rules -> reconcile ->
    cdi_emit_kind, four Allocate-shaped threads alloc_names_kind -> preferred_allocation (warp and large requests in
    one call) -> lw_encode_topo -> names; 10 rounds each, inputs picked by a per-thread seed from answers computed
    before the threads start.  Fails when calls interleave inside the context's lock, or when one caller's epochs
    or words leak into another's look-back."""
    redisc = [[cases.classify_rules(4097 + 1000 * v, 60 + v), cases.reconcile(1500 + 700 * v, 60 + v),
               cases.cdi_emit(200 + 300 * v, 60 + v, KIND)] for v in range(3)]
    alloc = [[cases.alloc_names(4096 + 2000 * v, 70 + v, KIND), cases.preferred_allocation(1 + v % 2, 2, 6, 70 + v),
              cases.lw_encode(5000 + 1000 * v, 70 + v, topo=True), cases.names(4500 + 1500 * v, 70 + v)] for v in range(3)]
    check_multi_tile([c for v in redisc + alloc for c in v])
    kx = fresh(KXPU_SCAN_EPOCH_LIMIT="5")
    tab, rows = load_names_table(kx, pci_text, oracle_rows)
    errors = []

    def worker(t):
        try:
            rng = np.random.default_rng(1000 + t)
            pool = redisc if t % 2 == 0 else alloc
            for r in range(10):
                for c in pool[int(rng.integers(0, len(pool)))]:
                    run(kx, c, "thread %d round %d" % (t, r), tab, rows)
        except Exception as e:  # noqa: BLE001
            errors.append("thread %d: %r" % (t, e))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    try:
        for th in threads:
            th.start()
        for th in threads:
            th.join()
    finally:
        tab.free()
    assert not errors, errors[:3]
