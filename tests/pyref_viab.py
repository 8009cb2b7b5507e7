"""Independent Python restatement of IOMMU group viability (include/kxpu.h, ABI v8), the second checker next to
oracle/kxpu_viab_oracle.c.  It walks the numpy records itself, with Python bytes and dicts: which groups come into
existence and in which order, then the first blocker of each.  It shares no code with the C oracle or the classify
checkers."""
BLOCKS, IS_DIR, VENDOR_ERR, DRIVER_ERR, IOMMU_ERR, DEVICE_ERR = 0x80, 0x10, 0x01, 0x02, 0x04, 0x08
VIABLE = 0xFFFFFFFF


def _id(txt, n):
    """readIDFromFile on the first n bytes: data[2:] with '\\n' trimmed at both ends; None when n is not 2..8."""
    if not 2 <= n <= 8:
        return None
    return bytes(txt[:n])[2:].strip(b"\n")


def is_candidate(rules, r):
    """A record some rule (vendor bytes, driver bytes) takes, with every read it needs working."""
    fl = int(r["flags"])
    if fl & (IS_DIR | VENDOR_ERR | DRIVER_ERR | IOMMU_ERR):
        return False
    vendor = _id(r["vendor_txt"], int(r["vendor_len"]))
    if vendor is None:
        return False
    return (vendor, bytes(r["driver"])) in set(rules)


def is_blocker(rules, r):
    fl = int(r["flags"])
    return bool(fl & BLOCKS) and not fl & IS_DIR and not is_candidate(rules, r)


def viability(rules, recs):
    """[(group id, first blocker or VIABLE)] in the order the groups come into existence; the string "unsupported"
    when a blocker carries group 0xFFFFFFFF."""
    first_blocker, groups, seen = {}, [], set()
    for i, r in enumerate(recs):
        g = int(r["iommu_group"])
        if is_blocker(rules, r):
            if g == 0xFFFFFFFF:
                return "unsupported"
            first_blocker.setdefault(g, i)
        elif is_candidate(rules, r) and g not in seen:
            # a group starts at a candidate whose device read works
            if not int(r["flags"]) & DEVICE_ERR and _id(r["device_txt"], int(r["device_len"])) is not None:
                groups.append(g)
                seen.add(g)
    return [(g, first_blocker.get(g, VIABLE)) for g in groups]
