"""Independent pure-Python restatement of the full pci.ids model (vendor, subsystem and class-section rows),
for small inputs.  Written from the file's own format statement (the header of tests/golden/pci.ids.gz):

    vendor  vendor_name
    \\t device  device_name                                  <-- single tab
    \\t\\t subvendor subdevice  subsystem_name                 <-- two tabs
    C class  class_name
    \\t subclass  subclass_name                               <-- single tab
    \\t\\t prog-if  prog-if_name                               <-- two tabs

with the reference's matching rules carried down to every level: ids are raw byte prefixes in lowercase hex, the
first line of an id wins (a vendor or class line in the file, a device or subclass line in its block, a subsystem or
prog-if line under its device or subclass line), comment lines do not end a block, and any other line that is not
indented (a blank line too) does.  Lines follow bufio.Scanner: a trailing '\\r' is dropped and the scan stops at the
first line of 64 KiB or more (pyref.scan_lines).  Shares no code with oracle/kxpu_oracle.c::kxo_full_build.

Rows are (key, offset of the line):
    kind 0  vendor     v
    kind 1  subsystem  v << 48 | d << 32 | sv << 16 | sd
    kind 2  class      1 << 24 | c << 16;  subclass 2 << 24 | c << 16 | s << 8;  prog-if 3 << 24 | c << 16 | s << 8 | p
"""
import re

from pyref import scan_lines

HEX4 = re.compile(rb"[0-9a-f]{4}")
HEX2 = re.compile(rb"[0-9a-f]{2}")
SUBSYS = re.compile(rb"([0-9a-f]{4}) ([0-9a-f]{4})")
CLASS = re.compile(rb"C ([0-9a-f]{2})")


def _id(pattern, line, at):
    """the hex id the pattern matches at line[at:], as an int, or None"""
    m = pattern.match(line, at)
    return None if m is None else int(m.group(0), 16)


def full_rows(text: bytes):
    """{kind: [(key, line offset), ...] in file order} for kinds 0, 1, 2."""
    rows = {0: [], 1: [], 2: []}
    vendors, classes = set(), set()
    block = None      # ("vendor", v, devices seen) / ("class", c, subclasses seen) / None
    parent = None     # the winning device / subclass line governing double-tab lines: (key prefix, keys seen) or None
    for off, line in scan_lines(text):
        if line.startswith(b"#"):
            continue
        if line.startswith(b"\t\t"):
            if parent is None:
                continue
            prefix, seen = parent
            if block[0] == "vendor":
                m = SUBSYS.match(line, 2)
                if m is None:
                    continue
                key, kind = prefix | int(m.group(1), 16) << 16 | int(m.group(2), 16), 1
            else:
                p = _id(HEX2, line, 2)
                if p is None:
                    continue
                key, kind = prefix | p, 2
            if key not in seen:
                seen.add(key)
                rows[kind].append((key, off))
            continue
        if line.startswith(b"\t"):
            parent = None
            if block is None:
                continue
            kind, top, seen = block
            if kind == "vendor":
                d = _id(HEX4, line, 1)
                if d is not None and d not in seen:
                    seen.add(d)
                    parent = (top << 48 | d << 32, set())
            else:
                s = _id(HEX2, line, 1)
                if s is not None and s not in seen:
                    seen.add(s)
                    rows[2].append((2 << 24 | top << 16 | s << 8, off))
                    parent = (3 << 24 | top << 16 | s << 8, set())
            continue
        # any other line is a top-level line: it ends the block, and may open one if it is the first of its id
        block = parent = None
        m = CLASS.match(line)
        if m is not None:
            c = int(m.group(1), 16)
            if c not in classes:
                classes.add(c)
                rows[2].append((1 << 24 | c << 16, off))
                block = ("class", c, set())
            continue
        v = _id(HEX4, line, 0)
        if v is not None and v not in vendors:
            vendors.add(v)
            rows[0].append((v, off))
            block = ("vendor", v, set())
    return rows


def full_build(text: bytes, kind: int):
    """rows of one kind, [(key, line offset), ...] in file order"""
    return full_rows(text)[kind]
