"""Plain-Python writer of kxpu_metrics_devices' document (include/kxpu.h) from the same records, and helpers that build
those records.  Label values are repaired with bytes.decode("utf-8", "replace") and then escaped (backslash, double
quote, LF), which is the rule the header states."""
import numpy as np

from kxpu_b200.binding import (METRICDEV_DTYPE, METRICREASON_DTYPE, METRICS_HEADS, METRICS_NO_VALUE, METRICS_REASONS)

NAMES = (b"kata_xpu_device_healthy", b"kata_xpu_device_unhealthy_reason", b"kata_xpu_pcie_aer_errors")


def label(raw: bytes) -> bytes:
    t = raw.decode("utf-8", "replace")
    return t.replace("\\", "\\\\").replace('"', '\\"').replace("\n", "\\n").encode()


def document(devs, strings: bytes, reasons) -> bytes:
    """families 1 to 3 of the metrics text of devs (METRICDEV_DTYPE) and reasons (METRICREASON_DTYPE)"""
    fam = [[], [], []]
    for d in devs:
        res = label(strings[int(d["resource_off"]):int(d["resource_off"]) + int(d["resource_len"])])
        addr = label(strings[int(d["address_off"]):int(d["address_off"]) + int(d["address_len"])])
        common = b'{resource="%s",device="%d",address="%s"' % (res, int(d["group"]), addr)
        fam[0].append(NAMES[0] + common + b"} %d\n" % int(d["healthy"]))
        for r in reasons[int(d["reason_off"]):int(d["reason_off"]) + int(d["reason_count"])]:
            detail = strings[int(r["detail_off"]):int(r["detail_off"]) + int(r["detail_len"])]
            fam[1].append(NAMES[1] + common + b',reason="%s",detail="%s"} 1\n' % (METRICS_REASONS[int(r["kind"])].encode(),
                                                                                   label(detail)))
        for sev, v in ((b"fatal", int(d["aer_fatal"])), (b"nonfatal", int(d["aer_nonfatal"]))):
            if v != METRICS_NO_VALUE:
                fam[2].append(NAMES[2] + common + b',severity="%s"} %d\n' % (sev, v))
    return b"".join(METRICS_HEADS[f] + b"".join(fam[f]) for f in range(3) if fam[f])


def counters(aer=0, cdev=0, sriov=0, reset=0, nvidia=0, live=0, snapshot=0) -> bytes:
    """family 4, the host's counters"""
    out = METRICS_HEADS[3]
    for f, v in (("aer_dev", aer), ("vfio-dev", cdev), ("sriov", sriov), ("reset", reset), ("nvidia", nvidia)):
        out += b'kata_xpu_sysfs_reads_total{file="%s"} %d\n' % (f.encode(), v)
    out += METRICS_HEADS[4]
    out += b'kata_xpu_allocate_validations_total{path="live"} %d\n' % live
    out += b'kata_xpu_allocate_validations_total{path="snapshot"} %d\n' % snapshot
    return out


class Builder:
    """devices in order: add(resource, group, address, healthy, [(kind, detail)], aer_fatal, aer_nonfatal)"""

    def __init__(self):
        self.strings = bytearray()
        self.devs, self.reasons = [], []

    def _put(self, b: bytes):
        off = len(self.strings)
        self.strings += b
        return off, len(b)

    def add(self, resource, group, address, healthy=1, reasons=(), aer_fatal=METRICS_NO_VALUE,
            aer_nonfatal=METRICS_NO_VALUE):
        ro, rl = self._put(resource)
        ao, al = self._put(address)
        r0 = len(self.reasons)
        for kind, detail in reasons:
            do, dl = self._put(detail)
            self.reasons.append((kind, dl, do))
        self.devs.append((ro, ao, rl, al, group, healthy, aer_fatal, aer_nonfatal, r0, len(reasons), 0))
        return self

    def arrays(self):
        return (np.array(self.devs, METRICDEV_DTYPE), bytes(self.strings), np.array(self.reasons, METRICREASON_DTYPE))
