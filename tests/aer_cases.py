"""Files for the AER tests (kxpu_aer_health, ABI v12) in the kernel's aer_dev_fatal / aer_dev_nonfatal format, with the
count each one must give, and the taint tables of the _taints tests."""
import numpy as np

from kxpu_b200.workloads import aer_file

UNKNOWN = (1 << 64) - 1
F, N = "TOTAL_ERR_FATAL", "TOTAL_ERR_NONFATAL"


def _pad_to(total_name, size, count=7):
    """a file of exactly `size` bytes whose last line is the TOTAL line with `count`"""
    tail = ("%s %d\n" % (total_name, count)).encode()
    body = b""
    while len(body) + len(tail) < size:
        line = b"Padding kind %d\n" % len(body)
        body += line if len(body) + len(line) + len(tail) <= size else b"x" * (size - len(body) - len(tail) - 1) + b"\n"
    return body + tail


def cases(total_name):
    """[(name, file bytes, count)] for the fatal (total_name = F) or non-fatal (N) file"""
    p = total_name + " "
    other = N if total_name == F else F
    c = [
        ("zero", aer_file(total_name, [0] * 18), 0),
        ("two", aer_file(total_name, [0, 1] + [0] * 15 + [1]), 2),
        ("names with spaces", ("Data Link Protocol 1\nSurprise Down Error 3\n%s4\n" % p).encode(), 4),
        ("total not last", ("%s5\nTLP 5\nDLP 0\n" % p).encode(), 5),
        ("two totals", ("%s5\nTLP 0\n%s9\n" % (p, p)).encode(), 9),
        ("last total bad", ("%s5\n%s09\n" % (p, p)).encode(), UNKNOWN),
        ("no newline", ("TLP 3\n%s3" % p).encode(), 3),
        ("prefix X", ("%sX 3\n" % total_name).encode(), UNKNOWN),
        ("prefix X then good", ("%s1\n%sX 3\n" % (p, total_name)).encode(), 1),
        ("other total", ("%s 3\n" % other).encode(), UNKNOWN),
        ("not at line start", ("x %s3\n" % p).encode(), UNKNOWN),
        ("cr", ("%s3\r\n" % p).encode(), UNKNOWN),
        ("leading zero", ("%s007\n" % p).encode(), UNKNOWN),
        ("zero alone", ("%s0" % p).encode(), 0),
        ("double zero", ("%s00\n" % p).encode(), UNKNOWN),
        ("empty number", ("%s\n" % p).encode(), UNKNOWN),
        ("two spaces", ("%s 5\n" % p).encode(), UNKNOWN),
        ("trailing space", ("%s5 \n" % p).encode(), UNKNOWN),
        ("sign", ("%s+5\n" % p).encode(), UNKNOWN),
        ("2^64-2", ("%s%d\n" % (p, (1 << 64) - 2)).encode(), (1 << 64) - 2),
        ("2^64-1", ("%s%d\n" % (p, (1 << 64) - 1)).encode(), UNKNOWN),
        ("2^64", ("%s%d\n" % (p, 1 << 64)).encode(), UNKNOWN),
        ("20 digits", ("%s%d\n" % (p, 10 ** 19)).encode(), 10 ** 19),
        ("21 digits", ("%s%d\n" % (p, 10 ** 20)).encode(), UNKNOWN),
        ("99...9 (20)", ("%s%s\n" % (p, "9" * 20)).encode(), UNKNOWN),
        ("empty", b"", UNKNOWN),
        ("only newlines", b"\n\n\n", UNKNOWN),
        ("4096 bytes", _pad_to(total_name, 4096), 7),
        ("4097 bytes", _pad_to(total_name, 4097), UNKNOWN),
        ("NUL in number", ("%s1\x002\n" % p).encode(), UNKNOWN),
        ("high bytes", b"\xff\xfe " + ("\n%s8\n" % p).encode(), 8),
    ]
    # the TOTAL line at every phase of the 32-byte windows the kernel walks
    for k in range(0, 70, 3):
        c.append(("pad %d" % k, b"y" * k + ("\n%s%d\n" % (p, k)).encode() + b"z" * (k % 5), k))
    return c


def pack(files, gaps=None, share=None):
    """(text, file_off [2n], file_len [2n]) for pairs files = [(fatal bytes, nonfatal bytes)]: each file after a gap of
    gaps[j] bytes (1..7 by default, so offsets are unaligned); share[i] = j makes record i use record j's files"""
    text, off, ln = b"", [], []
    for j, pair in enumerate(files):
        for f in pair:
            text += b"#" * (gaps[2 * j] if gaps is not None else 1 + (len(off) * 5) % 7)
            off.append(len(text))
            ln.append(len(f))
            text += f
    off, ln = np.array(off, np.uint64), np.array(ln, np.uint32)
    if share is not None:
        idx = np.repeat(np.asarray(share), 2) * 2 + np.tile([0, 1], len(share))
        off, ln = off[idx], ln[idx]
    return text, off, ln


# taint tables of the _taints calls
DRV = "vfio.nvidia.com"
TABLE3 = [(DRV + "/unhealthy", "vfio-device-missing", "NoSchedule"), (DRV + "/pcie-aer", "fatal", "NoSchedule"),
          (DRV + "/pcie-aer", "nonfatal", "NoSchedule")]


def long_table(k):
    """k entries at the longest key and value, distinct keys"""
    from dra_taint_cases import LONG_KEY, LONG_VALUE
    return [(LONG_KEY[:-2] + "%dZ" % t, LONG_VALUE, "NoSchedule" if t % 2 else "NoExecute") for t in range(k)]


def since_table(n, k, seed=0, frac=3, table=None):
    """int64 [n, k]: each entry carried with probability 1/frac at a random time, otherwise one of several negative
    values; with `table`, a device never carries two entries with one key and effect"""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 253402300799 + 1, (n, k), dtype=np.int64)
    neg = rng.choice(np.array([-1, -2, -(1 << 40), -(1 << 63)], np.int64), (n, k))
    s = np.where(rng.integers(0, frac, (n, k)) == 0, t, neg)
    if table is not None:
        for a in range(k):
            for b in range(a):
                if table[a][0] == table[b][0] and table[a][2] == table[b][2]:
                    s[:, a] = np.where(s[:, b] >= 0, -1, s[:, a])
    return s
