"""Independent Python restatement of kxpu_reconcile (include/kxpu.h, ABI v6), the second checker next to
oracle/kxpu_reconcile_oracle.c: two dicts keyed by the key bytes, one pass over cur in walk order."""
RC_KEPT, RC_NEW, RC_CHANGED, RC_RETIRED = 0, 1, 2, 3


def key_valid(key: bytes) -> bool:
    """The 40 key bytes (NUL padded as numpy's S40 strips them back to `key`): non-empty and no byte after a NUL."""
    return len(key) > 0 and b"\0" not in key


def reconcile(prev, cur, next_index):
    """prev / cur: lists of (key bytes, group, klass, tag, index).  Returns dict(index, cur_state, prev_state, counts)
    or None when the input is invalid."""
    if next_index + len(cur) >= 1 << 64:
        return None
    by_key = {}
    for j, (k, g, c, t, idx) in enumerate(prev):
        if not key_valid(k) or idx >= next_index or k in by_key:
            return None
        by_key[k] = j
    seen = set()
    for e in cur:
        if not key_valid(e[0]) or e[0] in seen:
            return None
        seen.add(e[0])
    prev_state = [RC_RETIRED] * len(prev)
    index, cur_state = [], []
    nxt = next_index
    for k, g, c, t, _ in cur:
        j = by_key.get(k)
        if j is not None and prev[j][1:4] == (g, c, t):
            st = RC_KEPT
            index.append(prev[j][4])
        else:
            st = RC_NEW if j is None else RC_CHANGED
            index.append(nxt)
            nxt += 1
        cur_state.append(st)
        if j is not None:
            prev_state[j] = st
    kept = cur_state.count(RC_KEPT)
    changed = cur_state.count(RC_CHANGED)
    counts = dict(n_kept=kept, n_new=cur_state.count(RC_NEW), n_changed=changed,
                  n_retired=prev_state.count(RC_RETIRED), next_index_out=nxt)
    return dict(index=index, cur_state=cur_state, prev_state=prev_state, counts=counts)


def rows(arr):
    """A SNAPREC_DTYPE array as the tuples reconcile() takes."""
    return [(bytes(r["key"]), int(r["iommu_group"]), int(r["klass"]), int(r["tag"]), int(r["index"])) for r in arr]
