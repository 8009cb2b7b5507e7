"""Taint arguments for the DRA taint tests (kxpu_dra_slices_taint / kxpu_dra_slices_mdev_taint, ABI v11): the longest
key and value, the timestamp edges, seeded taint patterns and the refused arguments."""
import numpy as np

KEY = "vfio.nvidia.com/unhealthy"
VALUE = "vfio-device-missing"
# the longest key (127 bytes: a 63-byte prefix, '/', a 63-byte name) and value (63 bytes)
LONG_KEY = "p" * 30 + "." + "q" * 32 + "/" + "N" + ("a-b_c.d" * 9)[:61] + "Z"
LONG_VALUE = "V" + ("x_y-z.w" * 9)[:61] + "0"
assert len(LONG_KEY) == 127 and len(LONG_VALUE) == 63
SINCE_MAX = 253402300799
# unix time -> timeAdded: the epoch, 2000-02-29 (a leap day of a 400-year century), 2100-03-01 (2100 is not a leap
# year), the last second of year 9999, and the seconds around them
EDGES = {
    0: "1970-01-01T00:00:00Z",
    951782400: "2000-02-29T00:00:00Z",
    951868799: "2000-02-29T23:59:59Z",
    951868800: "2000-03-01T00:00:00Z",
    4107542399: "2100-02-28T23:59:59Z",
    4107542400: "2100-03-01T00:00:00Z",
    1767225599: "2025-12-31T23:59:59Z",
    SINCE_MAX: "9999-12-31T23:59:59Z",
}


def since_pattern(n, kind, seed=0):
    """int64 taint times for n devices: kind "none" (all -1), "some" (about one in three tainted, negative values of
    several sizes for the rest), "all" (every device tainted), "edges" (the EDGES times in turn)"""
    rng = np.random.default_rng(seed)
    if kind == "none":
        return np.full(n, -1, np.int64)
    if kind == "edges":
        e = np.array(sorted(EDGES), np.int64)
        return e[np.arange(n) % len(e)]
    t = rng.integers(0, SINCE_MAX + 1, n, dtype=np.int64)
    if kind == "all":
        return t
    neg = rng.choice(np.array([-1, -2, -(1 << 40), -(1 << 63)], np.int64), n)
    return np.where(rng.integers(0, 3, n) == 0, t, neg)


# (key, value, effect) the calls refuse with KXPU_E_INVALID when taint_since is given
INVALID = [
    ("", VALUE, "NoSchedule"),
    (None, VALUE, "NoSchedule"),
    (LONG_KEY + "x", VALUE, "NoSchedule"),                  # 128 bytes
    ("p" * 64 + "/x", VALUE, "NoSchedule"),                 # a prefix label of 64 bytes
    ("Example.com/x", VALUE, "NoSchedule"),                 # an uppercase prefix
    ("/unhealthy", VALUE, "NoSchedule"),                    # an empty prefix
    ("example.com/", VALUE, "NoSchedule"),                  # an empty name
    ("a/b/c", VALUE, "NoSchedule"),
    ("example.com/-x", VALUE, "NoSchedule"),
    ("example.com/x_", VALUE, "NoSchedule"),
    ("example.com/" + "n" * 64, VALUE, "NoSchedule"),
    ("un healthy", VALUE, "NoSchedule"),
    ('un"healthy', VALUE, "NoSchedule"),
    (KEY, None, "NoSchedule"),
    (KEY, "-missing", "NoSchedule"),
    (KEY, "missing.", "NoSchedule"),
    (KEY, "v" * 64, "NoSchedule"),
    (KEY, "a/b", "NoSchedule"),
    (KEY, VALUE, "PreferNoSchedule"),
    (KEY, VALUE, "noschedule"),
    (KEY, VALUE, "NoSchedule "),
    (KEY, VALUE, ""),
    (KEY, VALUE, None),
]
