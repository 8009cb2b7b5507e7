"""Independent Python restatement of the NUMA topology calls (include/kxpu.h, ABI v5), the second checker next to
oracle/kxpu_topo_oracle.c:
  - group_masks: the masks from a plain walk over the records and the classify output's busIndex / group ids;
  - lw_bytes: the ListAndWatchResponse from google.protobuf messages declared at runtime (v1beta1 Device /
    TopologyInfo / NUMANode), serialised deterministically;
  - preferred: the allocation as one sorted() with key (bin rank, position).
"""
import numpy as np
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

NUMA_FLAG = 64


def record_numa(rec):
    """The node of one record (kxpu_devrec or kxpu_mdevrec row), or None."""
    if int(rec["flags"]) & NUMA_FLAG and int(rec["reserved0"]) < 64:
        return int(rec["reserved0"])
    return None


def group_masks(recs, res):
    """group_numa from a walk: every accepted record (accept_index != REJECTED) ORs its node into its group's mask;
    the masks are then listed in res["group_ids"] order."""
    by_group = {}
    for i in range(len(recs)):
        if int(res["accept_index"][i]) == 0xFFFFFFFF:
            continue
        g = int(recs[i]["iommu_group"])
        k = record_numa(recs[i])
        by_group[g] = by_group.get(g, 0) | ((1 << k) if k is not None else 0)
    return np.array([by_group.get(int(g), 0) for g in res["group_ids"]], np.uint64)


# ---------------------------------------------------------------- v1beta1 messages, declared at runtime
_CLASSES = None


def _classes():
    global _CLASSES
    if _CLASSES is None:
        fd = descriptor_pb2.FileDescriptorProto(name="kxpu_topo_v1beta1.proto", package="v1beta1", syntax="proto3")
        F = descriptor_pb2.FieldDescriptorProto

        def msg(name, fields):
            m = fd.message_type.add(name=name)
            for fname, num, typ, label, tname in fields:
                f = m.field.add(name=fname, number=num, type=typ, label=label)
                if tname:
                    f.type_name = tname

        opt, rep = F.LABEL_OPTIONAL, F.LABEL_REPEATED
        msg("NUMANode", [("ID", 1, F.TYPE_INT64, opt, None)])
        msg("TopologyInfo", [("nodes", 1, F.TYPE_MESSAGE, rep, ".v1beta1.NUMANode")])
        msg("Device", [("ID", 1, F.TYPE_STRING, opt, None), ("health", 2, F.TYPE_STRING, opt, None),
                       ("topology", 3, F.TYPE_MESSAGE, opt, ".v1beta1.TopologyInfo")])
        msg("ListAndWatchResponse", [("devices", 1, F.TYPE_MESSAGE, rep, ".v1beta1.Device")])
        pool = descriptor_pool.DescriptorPool()
        pool.Add(fd)
        _CLASSES = {n: message_factory.GetMessageClass(pool.FindMessageTypeByName("v1beta1." + n))
                    for n in ("NUMANode", "TopologyInfo", "Device", "ListAndWatchResponse")}
    return _CLASSES


def lw_message(groups, healthy=None, masks=None):
    M = _classes()
    resp = M["ListAndWatchResponse"]()
    for i, g in enumerate(groups):
        d = resp.devices.add()
        d.ID = str(int(g))
        d.health = "Healthy" if healthy is None or healthy[i] else "Unhealthy"
        m = int(masks[i]) if masks is not None else 0
        if m:
            d.topology.SetInParent()
            for k in range(64):
                if (m >> k) & 1:
                    d.topology.nodes.add().ID = k
    return resp


def lw_bytes(groups, healthy=None, masks=None) -> bytes:
    return lw_message(groups, healthy, masks).SerializeToString(deterministic=True)


def lw_parse(b: bytes):
    """[(ID, health, [nodes])] of a ListAndWatchResponse."""
    resp = _classes()["ListAndWatchResponse"]()
    resp.ParseFromString(b)
    return [(d.ID, d.health, [n.ID for n in d.topology.nodes]) for d in resp.devices]


# ---------------------------------------------------------------- preferred allocation
def _home(m):
    m = int(m)
    return (m & -m).bit_length() - 1 if m else 64


def preferred(dev_numa, requests):
    """[(available, must-include, size)] -> one position list per request, or None when any request is invalid."""
    out = []
    for avail, must, size in requests:
        avail, must = [int(x) for x in avail], [int(x) for x in must]
        n = len(dev_numa)
        if (any(p >= n for p in avail + must) or len(set(avail)) != len(avail) or len(set(must)) != len(must)
                or not set(must) <= set(avail) or size < len(must) or size > len(avail)):
            return None
        U = {_home(dev_numa[p]) for p in must} - {64}
        cands = [p for p in avail if p not in set(must)]
        c = {}
        for p in cands:
            c[_home(dev_numa[p])] = c.get(_home(dev_numa[p]), 0) + 1

        def bin_rank(k):
            return (2 if k == 64 else (0 if k in U else 1), -c.get(k, 0), k)
        pick = sorted(cands, key=lambda p: (bin_rank(_home(dev_numa[p])), p))
        out.append(must + pick[:size - len(must)])
    return out
