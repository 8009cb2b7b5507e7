"""Independent Python restatement of kxpu_reset_check (include/kxpu.h, an addition to ABI v14), the second checker next
to tests/reset_oracle.c: reset_method with bytes.split, the chains from pyref_pcie's regular expressions, and each
bridge's set S(B) built as a dict from bridge key to the list of records below it."""
import pyref_pcie as PP

NAMES = (b"flr", b"af_flr", b"pm", b"bus", b"cxl_bus", b"device_specific", b"acpi")
FILE_MAX = 64
ABSENT, READ_ERR, LEGACY = 1, 2, 4
ALL, UNNAMED = 0x7F, 0x80
SET_OK, NO_PATH, ROOT_BUS = 0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFFD
VIABLE = 0xFFFFFFFF
HOST_BRIDGE = 1 << 63
DRIVER_ERR, IOMMU_ERR, IS_DIR = 0x02, 0x04, 0x10


def methods(txt: bytes, length: int, flags: int) -> int:
    if flags & READ_ERR or length > FILE_MAX:
        return 0
    if flags & ABSENT:
        return UNNAMED if flags & LEGACY else 0
    t = txt[:length]
    if t.endswith(b"\n"):
        t = t[:-1]
    return sum(1 << k for k, name in enumerate(NAMES) if name in t.split(b" "))


def function_reset(m: int, allow: int) -> bool:
    return bool(m & allow) or (bool(m & UNNAMED) and allow == ALL)


def reset_check(rules, recs, paths, rrs, allow, group_off, group_members):
    """dict(methods, set_verdict, group_reset) as lists, or None for an invalid CSR."""
    n, G = len(recs), len(group_off) - 1
    for g in range(G):
        if group_off[g + 1] < group_off[g] or any(int(m) >= n for m in group_members[group_off[g]:group_off[g + 1]]):
            return None
    drivers = {bytes(d).rstrip(b"\0") for _, d in rules}
    bound = [bytes(r["driver"]).split(b"\0", 1)[0] in drivers and not int(r["flags"]) & (DRIVER_ERR | IOMMU_ERR | IS_DIR)
             for r in recs]
    meth = [methods(bytes(s["txt"]), int(s["len"]), int(s["flags"])) for s in rrs]
    chain = [PP.record_chain(recs[i], paths[i]) for i in range(n)]
    below = {}
    for j in range(n):
        for k in set(chain[j]):
            if not k & HOST_BRIDGE:
                below.setdefault(k, []).append(j)
    group = [int(r["iommu_group"]) for r in recs]
    verdict = []
    for i in range(n):
        if not chain[i]:
            verdict.append(NO_PATH)
            continue
        b = chain[i][-1]
        if b & HOST_BRIDGE:
            verdict.append(ROOT_BUS)
            continue
        s = below[b]
        unbound = [j for j in s if not bound[j]]
        groups = {group[j] for j in s}
        if unbound:
            verdict.append(min(unbound))
        elif groups == {group[i]}:
            verdict.append(SET_OK)
        else:
            want = min(groups) if group[i] != min(groups) else max(groups)
            verdict.append(min(j for j in s if group[j] == want))
    out = []
    for g in range(G):
        stuck = [int(i) for i in group_members[group_off[g]:group_off[g + 1]]
                 if not function_reset(meth[int(i)], allow) and verdict[int(i)] != SET_OK]
        out.append(min(stuck) if stuck else VIABLE)
    return dict(methods=meth, set_verdict=verdict, group_reset=out)
