"""Independent Python restatement of kxpu_dra_slices_taint / kxpu_dra_slices_mdev_taint (include/kxpu.h, ABI v11), the
second checker next to oracle/kxpu_dra_taint_oracle.c: each device dict of the v9 / v10 restatements gets a "taints"
list whose timeAdded comes from datetime, and the slices are written with json.dumps(..., separators=(",", ":")).
Argument and domain checks are the header's, in its order."""
import datetime
import json
import re

import pyref_dra
import pyref_dra_mdev
from pyref_dra import MAX_DEVICES, subdomain_ok

TAINT_SLICE = 64
SINCE_MAX = 253402300799
_NAME = re.compile(r"[A-Za-z0-9]([-A-Za-z0-9_.]*[A-Za-z0-9])?\Z")
EFFECTS = ("NoSchedule", "NoExecute")


def _s(x):
    if isinstance(x, bytes):
        try:
            return x.decode("ascii")
        except UnicodeDecodeError:
            return None
    return x


def key_ok(key):
    key = _s(key)
    if key is None or not 0 < len(key) <= 127:
        return False
    prefix, slash, name = key.rpartition("/")
    if slash and not subdomain_ok(prefix, 253):
        return False
    return len(name) <= 63 and bool(_NAME.match(name))


def value_ok(value):
    value = _s(value)
    return value is not None and (value == "" or (len(value) <= 63 and bool(_NAME.match(value))))


def time_added(since):
    return datetime.datetime.fromtimestamp(since, datetime.timezone.utc).strftime("%Y-%m-%dT%H:%M:%SZ")


def _slices(ref, driver, pool, node, generation, devs, key, value, effect, since):
    if since is None:
        return ref.slices(driver, pool, node, generation, devs)
    if not (subdomain_ok(driver, 63) and subdomain_ok(pool, 253) and subdomain_ok(node, 253) and 0 <= generation < 1 << 63):
        return -1
    if not (key_ok(key) and value_ok(value) and _s(effect) in EFFECTS):
        return -1
    if len(devs) >= MAX_DEVICES:
        return -7, None
    for r, t in zip(devs, since):
        w = ref.why(r) or ("taint_since" if int(t) > SINCE_MAX else None)
        if w:
            return -7, w
    driver, pool, node, key, value, effect = (_s(x) for x in (driver, pool, node, key, value, effect))
    taint = {"key": key}
    if value:
        taint["value"] = value
    taint["effect"] = effect
    count = max(1, -(-len(devs) // TAINT_SLICE))
    out, offs = b"", []
    for s in range(count):
        devices = []
        for r, t in zip(devs[s * TAINT_SLICE:(s + 1) * TAINT_SLICE], since[s * TAINT_SLICE:(s + 1) * TAINT_SLICE]):
            d = ref.device(r)
            if int(t) >= 0:
                d["taints"] = [dict(taint, timeAdded=time_added(int(t)))]
            devices.append(d)
        obj = {"kind": "ResourceSlice", "apiVersion": "resource.k8s.io/v1",
               "metadata": {"generateName": "%s-%s-" % (node, driver)},
               "spec": {"driver": driver, "pool": {"name": pool, "generation": generation, "resourceSliceCount": count},
                        "nodeName": node, "devices": devices}}
        offs.append(len(out))
        out += json.dumps(obj, separators=(",", ":")).encode() + b"\n"
    offs.append(len(out))
    return out, offs


def slices(driver, pool, node, generation, devs, key, value, effect, since):
    """kxpu_dra_slices_taint: (bytes, slice_off), or -1 (bad argument), or (-7, reason) as the oracle returns them"""
    return _slices(pyref_dra, driver, pool, node, generation, devs, key, value, effect, since)


def slices_mdev(driver, pool, node, generation, devs, key, value, effect, since):
    """kxpu_dra_slices_mdev_taint, the same way"""
    return _slices(pyref_dra_mdev, driver, pool, node, generation, devs, key, value, effect, since)
