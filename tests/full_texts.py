"""Edge texts of the full pci.ids model (subsystem rows and the class section), shared by the oracle tests
(pyref_full vs kxo_full_build) and the GPU parity tests (test_gpu_full.py)."""
import numpy as np

CW = 2048           # the chunk the full-model kernels give one warp
MAX_TOKEN = 65536   # bufio.Scanner stops at the first line this long

EDGE_TEXTS = [
    b"", b"\n", b"\t\t1234 5678  orphan\n",
    b"1234  V\n\t0001  d\n\t\t1111 2222  s\n\t\t1111 2222  dup\n\t0001  dupdev\n\t\t3333 4444  lost\n",
    b"C 01  cls\n\t02  sub\n\t\t03  pi\n\t\t03  dup\n\t02  dupsub\n\t\t04  lost\nC 01  again\n\t05  lost\n",
    b"1234  V\n\t0001  d\n#c\n\t\t1111 2222  after comment\n\n\t\t5555 6666  after blank\n",
    b"1234  V\r\n\t0001  d\r\n\t\t1111 2222  crlf\r\n", b"C 0g  bad\n\t01  x\n1234  V\n\t00  short\n\t\t1111 2222  under short\n",
    b"1234  V\n\t0001  d\n\t\t1111  one id only\n\t\t11112222  no blank\n\t\t1111 222  short\n\t\t1111 2222\n",
    # lowercase hex only: uppercase ids are no ids, and an uppercase vendor line still ends the block before it
    b"ABCD  upper\n\t0001  d\n\t\t1111 2222  s\nabcd  V\n\tFFFF  upper dev\n\t\t1111 2222  lost\n\tffff  dev\n"
    b"\t\tFFFF 0000  upper\n\t\tffff 0000  s\nC FF  upper\n\t01  lost\nC ff  cls\n\tFF  upper\n\t\t01  lost\n\tff  sub\n\t\tFF  x\n\t\tff  pi\n",
    # heads with too few digits at every level, raw prefixes, a line of tabs
    b"abc\n\t0001  d\n\t\t1111 2222  lost\nabcd\n\t001\n\t\t1111 2222  lost\n\t0001\n\t\t1111 2222\n\t\t1111 2222x\n\t\t\t3333 4444\n"
    b"C 0\n\t01\n\t\t01\nC 01\n\t0\n\t\t02  lost\n\t02\n\t\t0\n\t\t03\n\t\t\t04\n\t\t04x\n\t\n\t\t\n",
    # CRLF blank line ends a block; a lone '\r' line too
    b"1234  V\r\n\t0001  d\r\n\r\n\t\t1111 2222  lost\r\nC 01  c\r\n\t02  s\r\n\r\n\t\t03  lost\r\n",
]

# the all-ones subsystem key ffff ffff under device ffff of vendor ffff, in front of and behind ordinary keys
ALL_ONES = b"ffff  Illegal\n\tffff  all\n\t\tffff ffff  ones\n\t\tffff fffe  x\n\t\t0000 0000  z\n"
ALL_ONES_KEYS = [(1 << 64) - 1, (1 << 64) - 2, 0xffffffff00000000]
ALL_ONES_OFFS = [25, 43, 58]


def home_slot(keys, lg):
    """home slot of 64-bit keys in the full model's 2^lg-slot subsystem table (Fibonacci hashing)"""
    keys = np.asarray(keys, np.uint64)
    return (keys * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(64 - lg)


def all_ones_first(n_keys=200000, seed=3):
    """The all-ones block first, then about n_keys distinct subsystem keys of vendor ffff (at most 50 000 per device
    line), and keys whose home slot is the all-ones key's own in tables of 2^17 and 2^19 slots: they probe through
    the slot an insert of ~0 as an ordinary key would have touched."""
    rng = np.random.default_rng(seed)
    parts = [ALL_ONES]
    for lg in (17, 19):
        dev = 0x10 + lg
        cand = (np.uint64(0xffff0000 | dev) << np.uint64(32)) | rng.integers(0, 1 << 32, 1 << 22, dtype=np.uint64)
        hit = np.unique(cand[home_slot(cand, lg) == home_slot([(1 << 64) - 1], lg)[0]])[:16]
        assert len(hit) >= 8
        parts.append(b"\t%04x  collide %d\n" % (dev, lg))
        parts += [b"\t\t%04x %04x  c\n" % ((int(k) >> 16) & 0xffff, int(k) & 0xffff) for k in hit]
    per_dev = 50000
    for d in range((n_keys + per_dev - 1) // per_dev):
        parts.append(b"\t%04x  bulk\n" % d)
        ids = np.unique(rng.integers(0, 1 << 32, per_dev + 100, dtype=np.uint64))[:per_dev]
        parts.append(b"".join(b"\t\t%04x %04x\n" % (int(k) >> 16, int(k) & 0xffff) for k in ids))
    return b"".join(parts)


def long_line(length, kind=b"#"):
    """one line of `length` bytes before its '\\n' (a trailing '\\r' counts): a comment, or a vendor line"""
    return kind + b"x" * (length - len(kind))


LONG_LENGTHS = [(MAX_TOKEN - 1, True), (MAX_TOKEN, False), (None, False)]  # None: 65 535 bytes + '\r' (65 536 with it)


def cutoff_texts():
    """[(text, uncut text, kept)]: a line at the 64 KiB limit between a device line and its subsystem lines, between a
    class line and its subclass, in front of the class section and as an unterminated last line.  `uncut` holds the
    same lines with the long one shortened to 16 bytes: every row a cut would hide."""
    out = []
    for length, kept in LONG_LENGTHS:
        for where in range(4):
            def body(ln):
                tail = b"5678  W\n\t0002  D2\n\t\t3333 4444  S\n"
                if where == 0:
                    return (b"1234  V\n\t0001  D\n" + ln + b"\n\t\t1111 2222  S\n\t\tffff ffff  S2\n"
                            + b"C 01  K\n\t02  SC\n\t\t03  PI\n" + tail)
                if where == 1:
                    return b"1234  V\n\t0001  D\n\t\t1111 2222  S\nC 01  K\n" + ln + b"\n\t02  SC\n\t\t03  PI\n" + tail
                if where == 2:
                    return b"1234  V\n\t0001  D\n\t\t1111 2222  S\n" + ln + b"\nC 01  K\n\t02  SC\n\t\t03  PI\n" + tail
                return b"1234  V\n\t0001  D\n\t\t1111 2222  S\nC 01  K\n\t02  SC\n\t\t03  PI\n" + tail + ln
            kind = b"abcd  " if where == 3 else b"#"
            ln = long_line(MAX_TOKEN - 1, kind) + b"\r" if length is None else long_line(length, kind)
            out.append((body(ln), body(long_line(16, kind)), kept))
    return out


def template(s):
    """every line kind once, ids made distinct by s (class-section ids by s mod 256): vendor, device (CRLF), subsystem,
    comment, subsystem after the comment, the 11-byte subsystem head with no name, blank line, orphan subsystem, class,
    subclass, prog-if (CRLF), comment, prog-if, CRLF blank line, orphan prog-if"""
    c = s & 0xff
    return (b"%04x  Vendor %d\n\t%04x  Device\r\n\t\t%04x %04x  Sub\n# comment\n\t\t%04x 0001  After comment\r\n\t\t%04x 0002\n"
            b"\n\t\t%04x 0003  orphan\nC %02x  Class\n\t%02x  Subclass\n\t\t%02x  Progif\r\n#c\n\t\t%02x  Progif two\n\r\n\t\t%02x  orphan\n"
            % (0x1000 + s, s, 0xa000 + s, s, 0xf000 + s, s, s, s, c, 255 - c, c, 255 - c, c ^ 0x5a))


def pad_to(cur, target):
    """comment lines (each < 1 KiB) that take a text of length cur to exactly length target (target - cur >= 2)"""
    n = target - cur
    assert n >= 2 or n == 0
    out = []
    while n:
        k = min(n, 1000)
        if n - k == 1:
            k -= 1
        out.append(b"#" + b"p" * (k - 2) + b"\n")
        n -= k
    return b"".join(out)


def seam_text():
    """The template once per 2 KiB chunk, shifted by one byte per chunk: every line head lands on every offset from 41
    in front of a chunk boundary to 41 behind it."""
    t0 = len(template(0))
    parts, n = [], 0
    for s in range(t0 + 83):
        start = (s + 1) * CW - t0 - 41 + s
        parts.append(pad_to(n, start))
        parts.append(template(s))
        n = start + len(parts[-1])
    return b"".join(parts)


def lookback_texts():
    """Governing lines exactly 31, 32, 33, 64 and 65 chunks in front of their rows, with only comments in between
    (chunks without a top-level or single-tab line): the vendor line alone, and the vendor + device line, far back;
    the same for class and subclass."""
    out = []
    for dist in (31, 32, 33, 64, 65):
        for both in (False, True):
            head = b"abcd  V\n" + (b"\t0001  D\n" if both else b"")
            rows = (b"" if both else b"\t0001  D\n") + b"\t\t1111 2222  S\n\t\tffff ffff  S2\n"
            t = head + pad_to(len(head), dist * CW + 7) + rows
            out.append(t)
            head = b"C 0c  K\n" + (b"\t03  SC\n" if both else b"")
            rows = (b"" if both else b"\t03  SC\n") + b"\t\t30  PI\n\t\tff  PI2\n"
            out.append(head + pad_to(len(head), dist * CW + 7) + rows)
    return out


def length_texts():
    """texts of 2048 k - 1, 2048 k and 2048 k + 1 bytes, ending in a newline or in an unterminated subsystem line"""
    out = []
    for k in (1, 2, 33):
        for d in (-1, 0, 1):
            n = k * CW + d
            for last in (b"\t\t1111 2222  end\n", b"\t\tabcd ef01"):
                head = template(7) + b"1234  V\n\t0001  D\n"
                out.append(head + pad_to(len(head), n - len(last)) + last)
    return out
