"""Small workload for compute-sanitizer runs (memcheck / racecheck / synccheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import kxpu_b200 as K
from kxpu_b200 import workloads as W
kx = K.Kxpu(0)
text = W.load_pci_ids()
copies = int(os.environ.get("COPIES", "3"))
tab = kx.pciids_load(text * copies)
keys, offs, rows = kx.table_export(tab)
r = kx.lookup(tab, W.cfg2_queries(keys))
names, _, _ = kx.names(tab, r)
print("rows", tab.rows, "hits", int((r >= 0).sum()))
recs = W.cfg3_records(keys, n=20000)
res = kx.classify(recs)
devs = W.cfg5_devices(3000)
print("classify", res["n_accepted"], "json", len(kx.cdi_emit(1, devs)), "yaml", len(kx.cdi_emit(0, devs)))
print("alloc", len(kx.alloc_names(devs["index"])[0]), "lw", len(kx.lw_encode(res["group_ids"][:100])))
# NUMA topology: classify masks (PCI and mdev), topology wire bytes, both preferred-allocation shapes
tres = kx.classify_topo([(b"10de", b"vfio-pci")], W.topo_records(keys, n=20000, nodes=4))
mres = kx.classify_topo(W.MDEV_RULES, W.topo_mdev_records(n=20000), mdev=True)
dn = W.topo_dev_numa(20000)
print("topo groups", tres["n_groups"], mres["n_groups"], "lw", len(kx.lw_encode_topo(tres["group_ids"], None, tres["group_numa"])),
      "pref", len(kx.preferred_allocation(dn, W.topo_requests(dn, n_req=300))),
      len(kx.preferred_allocation(dn, W.topo_requests(dn, n_req=1, avail=20000, size=5000, must_max=3))[0]))
# rediscovery: index reconciliation over PCI and UUID keys
for mdev in (False, True):
    prev, cur, ni = W.reconcile_pair(3, 20000, mdev=mdev)
    print("reconcile", kx.reconcile(prev, cur, ni)["counts"])
tab.free()
# zero-copy join: text, keys and rows in mapped pinned host memory
h_t, p1 = kx.pinned(len(text)); h_t[:] = np.frombuffer(text, np.uint8)
qq = W.cfg2_queries(keys)
h_q, p2 = kx.pinned(len(qq) * 4, np.uint32); h_q[:] = qq
h_r, p3 = kx.pinned(len(qq) * 4, np.int32)
tz, rz = kx.pciids_join(h_t, h_q, rows_out=h_r)
print("zero-copy join rows", tz.rows, "hits", int((rz >= 0).sum()))
tz.free()
for p in (p1, p2, p3):
    kx.pinned_free(p)
# sharded load + join, three contexts of one process on this GPU
m = K.KxpuMulti([0, 0, 0])
big = text * 2
q = W.cfg2_queries(keys)[:768]
shards, bufs = [], []
for r, (a, b) in enumerate(K.plan_shards(big, 3)):
    k2 = m.ctxs[r]
    d = k2.dev_alloc(max(b - a, 16)); k2.upload(d, np.frombuffer(big[a:b], np.uint8))
    dq, dr = k2.dev_alloc(256 * 4), k2.dev_alloc(768 * 4)
    k2.upload(dq, q[256 * r:256 * r + 256])
    shards.append(dict(d_text=d, n=b - a, global_base=a, d_keys=dq, nq=256, key_offset=256 * r, d_rows_all=dr))
    bufs.append((k2, d, dq, dr))
for rep in range(3):
    tabs = m.pciids_join(shards, 768)
    print("sharded rows", [t.rows for t in tabs], "hits", int((m.ctxs[0].download(shards[0]["d_rows_all"], 768 * 4, np.int32) >= 0).sum()))
    for t in tabs:
        t.free()
for k2, d, dq, dr in bufs:
    k2.dev_free(d); k2.dev_free(dq); k2.dev_free(dr)
m.close()
