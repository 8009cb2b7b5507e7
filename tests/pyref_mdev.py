"""Independent Python restatement of vGPU discovery (include/kxpu.h: kxpu_classify_mdev, kxpu_mdev_names,
kxpu_cdi_emit_mdev), written from the header's text, not from either C implementation.  Slow; for small inputs."""
import re

import pyref

_UUID = re.compile(rb"[0-9a-f]{8}-[0-9a-f]{4}-[0-9a-f]{4}-[0-9a-f]{4}-[0-9a-f]{12}\Z")


def uuid_ok(u: bytes) -> bool:
    return _UUID.match(u) is not None


def type_key(name: bytes) -> bytes:
    name = name.strip(b"\t\n\v\f\r ").replace(b" ", b"_")
    return re.sub(rb"[^A-Za-z0-9_.-]", b"", name)


def _read_id(txt: bytes):
    if len(txt) < 2 or len(txt) > 8:
        return None
    return txt[2:].strip(b"\n")


def rec_key(r) -> bytes:
    """r: a dict with the fields of kxpu_mdevrec (bytes trimmed to their lengths)."""
    if r["name_err"] or len(r["name"]) > 40:
        return b""
    return type_key(r["name"])


def classify_mdev(rules, recs):
    """rules: [(vendor, driver)]; recs: dicts uuid, vendor (file bytes), driver, group, name (file bytes), is_dir,
    vendor_err, driver_err, iommu_err, name_err.  Returns accept_index, groups [(gid, [members])],
    devs [(first record, rule, [gids])]."""
    accept, groups, gindex, devs, dindex, first_of = [], [], {}, [], {}, {}
    bus = 0
    for i, r in enumerate(recs):
        accept.append(None)
        if r["is_dir"] or r["vendor_err"] or r["driver_err"] or r["iommu_err"]:
            continue
        if not uuid_ok(r["uuid"]) or r["group"] == 0xFFFFFFFF:
            continue
        vid = _read_id(r["vendor"])
        if vid is None:
            continue
        rule = next((q for q, (v, d) in enumerate(rules) if v == vid and d == r["driver"]), None)
        if rule is None:
            continue
        key = rec_key(r)
        if key:
            first_of.setdefault(key, i)
        g = r["group"]
        if g not in gindex:
            if not key:
                continue
            gindex[g] = len(groups)
            groups.append((g, []))
            dk = (rule, first_of[key])
            if dk not in dindex:
                dindex[dk] = len(devs)
                devs.append((first_of[key], rule, []))
            devs[dindex[dk]][2].append(g)
        groups[gindex[g]][1].append(i)
        accept[i] = bus
        bus += 1
    return accept, groups, devs


def _frag_yaml(kind, d):
    bdf = d["parent"]
    q = b'"' + bdf + b'"' if pyref.BASE60.match(bdf.decode()) else bdf
    return (b'  - name: "%d"\n    annotations:\n      attach-pci: "true"\n      bdf: %s\n      cdi.k8s.io/vfio%d: %s=%d\n'
            b"      mdev: %s\n    containerEdits:\n      deviceNodes:\n        - path: /dev/vfio/%d\n"
            % (d["index"], q, d["group"], kind, d["index"], d["uuid"], d["group"]))


def cdi_yaml(kind: bytes, devs):
    head = b"cdiVersion: 0.6.0\nkind: " + kind + b"\n"
    if not devs:
        return head + b"devices: []\n"
    return head + b"devices:\n" + b"".join(_frag_yaml(kind, d) for d in devs)


def cdi_json(kind: bytes, devs):
    head = b'{\n  "cdiVersion": "0.6.0",\n  "kind": "' + kind + b'",\n'
    if not devs:
        return head + b'  "devices": null,\n  "containerEdits": {}\n}'
    frags = [(b'    {\n      "name": "%d",\n      "annotations": {\n        "attach-pci": "true",\n        "bdf": "%s",\n'
              b'        "cdi.k8s.io/vfio%d": "%s=%d",\n        "mdev": "%s"\n      },\n      "containerEdits": {\n'
              b'        "deviceNodes": [\n          {\n            "path": "/dev/vfio/%d"\n          }\n        ]\n      }\n    }'
              % (d["index"], d["parent"], d["group"], kind, d["index"], d["uuid"], d["group"])) for d in devs]
    return head + b'  "devices": [\n' + b",\n".join(frags) + b'\n  ],\n  "containerEdits": {}\n}'
