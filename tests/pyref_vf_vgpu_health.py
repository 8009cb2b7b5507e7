"""Independent Python restatement of kxpu_vf_vgpu_drift (include/kxpu.h, additions to ABI v14): each record's current type
by pyref_vf_vgpu.current (the restatement of kxpu_vf_vgpu_types' current-type rule), compared with the walk's, then a
scan of each group's members in order.  It shares no code with the kernel."""
import pyref_vf_vgpu as PV

SAME, CLEARED, CHANGED, BAD = 0, 1, 2, 3
STEADY = 0xFFFFFFFF


def vf_vgpu_drift(recs_vt, type_was, group_off, group_members):
    """dict(type_now, status_now, group_first) as lists, or None where the call returns KXPU_E_INVALID."""
    n = len(recs_vt)
    if any(b < a for a, b in zip(group_off, group_off[1:])) or any(m >= n for m in group_members[:group_off[-1]]):
        return None
    type_now, status = [], []
    for r, was in zip(recs_vt, type_was):
        was = int(was)
        if not int(r["flags"]) & PV.VT_READ:
            type_now.append(was)
            status.append(SAME)
            continue
        st, v = PV.current(r)
        if st == PV.BAD:
            type_now.append(0)
            status.append(BAD)
        else:
            type_now.append(v)
            status.append(SAME if v == was else CLEARED if v == 0 else CHANGED)
    first = []
    for g in range(len(group_off) - 1):
        drifted = [p for p, m in enumerate(group_members[group_off[g]:group_off[g + 1]]) if status[m] != SAME]
        first.append(drifted[0] if drifted else STEADY)
    return dict(type_now=type_now, status_now=status, group_first=first)
