"""Independent Python restatement of kxpu_aer_health and kxpu_dra_slices_taints / kxpu_dra_slices_mdev_taints
(include/kxpu.h, ABI v12), the second checker next to oracle/kxpu_aer_oracle.c.  Counts are parsed with str and re;
the slices are the v11 restatement's untainted 64-device slices read back with json.loads, the taint lists added to each
device dict and the slice written again with json.dumps."""
import json
import re

import numpy as np

import pyref_dra_taint as PT
from pyref_dra import MAX_DEVICES, subdomain_ok

UNKNOWN = (1 << 64) - 1
FILE_MAX = 4096
FATAL, NONFATAL, UNKNOWN_BIT = 1, 2, 4
_NUMBER = re.compile(r"(0|[1-9][0-9]{0,19})\Z")


def count(data, prefix):
    """the count of one file (bytes), UNKNOWN when unknown"""
    if len(data) == 0 or len(data) > FILE_MAX:
        return UNKNOWN
    hits = [line for line in data.decode("latin-1").split("\n") if line.startswith(prefix)]
    if not hits or not _NUMBER.match(hits[-1][len(prefix):]):
        return UNKNOWN
    v = int(hits[-1][len(prefix):])
    return v if v < UNKNOWN else UNKNOWN


def aer_health(text, file_off, file_len, fatal_limit, nonfatal_limit, group_off, group_members):
    """(totals, group_aer) or -1, as the oracle returns them"""
    n, G = len(file_off) // 2, len(group_off) - 1
    if any(int(group_off[g + 1]) < int(group_off[g]) for g in range(G)):
        return -1
    if any(int(o) > len(text) or int(l) > len(text) - int(o) for o, l in zip(file_off, file_len)):
        return -1
    members = [int(m) for m in group_members[int(group_off[0]):int(group_off[-1])]]
    if any(m >= n for m in members):
        return -1
    totals = [count(bytes(text[int(o):int(o) + int(l)]), "TOTAL_ERR_NONFATAL " if f % 2 else "TOTAL_ERR_FATAL ")
              for f, (o, l) in enumerate(zip(file_off, file_len))]
    aer = []
    for g in range(G):
        bits = 0
        for m in group_members[int(group_off[g]):int(group_off[g + 1])]:
            tf, tn = totals[2 * int(m)], totals[2 * int(m) + 1]
            bits |= (UNKNOWN_BIT if UNKNOWN in (tf, tn) else 0) | (FATAL if tf != UNKNOWN and tf > fatal_limit else 0)
            bits |= NONFATAL if tn != UNKNOWN and tn > nonfatal_limit else 0
        aer.append(bits)
    return np.array(totals, np.uint64), np.array(aer, np.uint8)


def _slices(one, ref, driver, pool, node, generation, devs, taints, since):
    if since is None:
        return ref.slices(driver, pool, node, generation, devs)
    if not (subdomain_ok(driver, 63) and subdomain_ok(pool, 253) and subdomain_ok(node, 253) and 0 <= generation < 1 << 63):
        return -1
    if not 0 < len(taints) <= 4 or not all(PT.key_ok(k) and PT.value_ok(v) and PT._s(e) in PT.EFFECTS for k, v, e in taints):
        return -1
    if len(devs) >= MAX_DEVICES:
        return -7, None
    since = np.asarray(since, np.int64).reshape(len(devs), len(taints))
    table = [tuple(PT._s(x) for x in t) for t in taints]
    for r, row in zip(devs, since):
        w = ref.why(r) or ("taint_since" if any(int(t) > PT.SINCE_MAX for t in row) else None)
        carried = [table[t] for t in range(len(table)) if row[t] >= 0]
        if not w and len({(k, e) for k, _, e in carried}) < len(carried):
            w = "taint_duplicate"
        if w:
            return -7, w
    # the untainted 64-device slices of the v11 call, then the lists added device by device
    blob, _ = one(driver, pool, node, generation, devs, table[0][0], table[0][1], table[0][2], np.full(len(devs), -1, np.int64))
    out, offs, i = b"", [], 0
    for line in blob.decode().splitlines():
        obj = json.loads(line)
        for d in obj["spec"]["devices"]:
            lst = []
            for (k, v, e), t in zip(table, since[i]):
                if t >= 0:
                    entry = {"key": k}
                    if v:
                        entry["value"] = v
                    entry.update(effect=e, timeAdded=PT.time_added(int(t)))
                    lst.append(entry)
            if lst:
                d["taints"] = lst
            i += 1
        offs.append(len(out))
        out += json.dumps(obj, separators=(",", ":")).encode() + b"\n"
    offs.append(len(out))
    return out, offs


def slices(driver, pool, node, generation, devs, taints, since):
    """kxpu_dra_slices_taints: (bytes, slice_off), or -1 (bad argument), or (-7, reason) as the oracle returns them"""
    import pyref_dra
    return _slices(PT.slices, pyref_dra, driver, pool, node, generation, devs, taints, since)


def slices_mdev(driver, pool, node, generation, devs, taints, since):
    """kxpu_dra_slices_mdev_taints, the same way"""
    import pyref_dra_mdev
    return _slices(PT.slices_mdev, pyref_dra_mdev, driver, pool, node, generation, devs, taints, since)
