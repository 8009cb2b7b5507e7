"""Small workload for compute-sanitizer runs (memcheck / racecheck / synccheck)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import kxpu_b200 as K
from kxpu_b200 import binding as B, workloads as W
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
# the vGPU cdev layout: 3000 mdevs with cdev numbers of every width, emitted and parsed back
mcd = np.zeros(3000, B.MDEVCDEV_DTYPE)
mcd["dev"], mcd["vfio_cdev"] = W.mdev_devices(3000), (np.arange(3000, dtype=np.uint64) * 1431655765) % (1 << 32)
for fmt_ in (0, 1):
    mdoc = kx.cdi_emit_mdev_cdev(fmt_, mcd, "nvidia.com/vgpu")
    assert kx.cdi_parse_mdev_cdev(fmt_, mdoc, "nvidia.com/vgpu").tobytes() == mcd.tobytes()
    print("mdev cdev spec", fmt_, len(mdoc))
# the typed VF-vGPU layouts: 3000 VFs with their vGPU types, emitted and parsed back in both node layouts
vcd = W.vf_vgpu_cdi_devices(3000)
for fmt_ in (0, 1):
    for cdev in (False, True):
        vdoc = kx.cdi_emit_vf_vgpu(fmt_, vcd, "nvidia.com/vgpu", cdev=cdev)
        got = kx.cdi_parse_vf_vgpu(fmt_, vdoc, "nvidia.com/vgpu", cdev=cdev)
        want = vcd.copy()
        if not cdev:
            want["dev"]["reserved"] = 0  # the group layout carries no cdev number
        assert got.tobytes() == want.tobytes()
        print("vf vgpu spec", fmt_, cdev, len(vdoc))
# NUMA topology: classify masks (PCI and mdev), topology wire bytes, both preferred-allocation shapes
tres = kx.classify_topo([(b"10de", b"vfio-pci")], W.topo_records(keys, n=20000, nodes=4))
mres = kx.classify_topo(W.MDEV_RULES, W.topo_mdev_records(n=20000), mdev=True)
dn = W.topo_dev_numa(20000)
print("topo groups", tres["n_groups"], mres["n_groups"], "lw", len(kx.lw_encode_topo(tres["group_ids"], None, tres["group_numa"])),
      "pref", len(kx.preferred_allocation(dn, W.topo_requests(dn, n_req=300))),
      len(kx.preferred_allocation(dn, W.topo_requests(dn, n_req=1, avail=20000, size=5000, must_max=3))[0]))
# PCIe topology: the forest of a walk, both preferred-allocation shapes over it
precs, ppaths, poff, pmem = W.pcie_walk(20000, group_max=1)
ptree = kx.pcie_tree(precs, ppaths, poff, pmem)
pnode = ptree["group_node"][:15000].copy()
pdn = W.topo_dev_numa(len(pnode))
print("pcie nodes", len(ptree["key"]), "pref",
      len(kx.preferred_allocation_pcie(pdn, pnode, ptree["parent"], ptree["depth"], W.topo_requests(pdn, n_req=300))),
      len(kx.preferred_allocation_pcie(pdn, pnode, ptree["parent"], ptree["depth"],
                                       W.topo_requests(pdn, n_req=1, avail=len(pnode), size=5000, must_max=3))[0]))
# one large PCIe request over 3 tiles + 1 position with r on the first tile seam: roots of 2048 positions, leaves of 16
# (776 nodes, so k_pick runs 4 CTAs), one home; size 4096 fits no node, so the answer is positions 0 .. 4095
sn = 3 * 4096 + 1
snode = (sn // 2048 + 1 + np.arange(sn) // 16).astype(np.uint32)
spar = np.concatenate([np.full(sn // 2048 + 1, B.PCIE_NO_NODE), np.arange(sn // 16 + 1) * 16 // 2048]).astype(np.uint32)
sdep = np.concatenate([np.zeros(sn // 2048 + 1), np.ones(sn // 16 + 1)]).astype(np.uint8)
seam = kx.preferred_allocation_pcie(np.ones(sn, np.uint64), snode, spar, sdep, [(np.arange(sn)[::-1].copy(), [], 4096)])[0]
assert seam == list(range(4096)) and len(spar) > 3 * 256
print("pcie seam request", len(seam), "nodes", len(spar))
# rediscovery: index reconciliation over PCI and UUID keys
for mdev in (False, True):
    prev, cur, ni = W.reconcile_pair(3, 20000, mdev=mdev)
    print("reconcile", kx.reconcile(prev, cur, ni)["counts"])
# IOMMU group viability: the blocker pass with and without NUMA masks
vrecs = W.viab_records(20000)
for topo in (False, True):
    vres = kx.classify_viable(W.VIAB_RULES, vrecs, topo=topo)
    print("viable groups", vres["n_groups"], "blocked", int((vres["group_blocker"] != B.VIABLE).sum()))
# SR-IOV: the verdict of a walk with PFs and VFs, and the forest with VFs below their PFs
srecs, ssrs = W.sriov_walk(20000)
sres = kx.classify_rules([(b"10de", b"vfio-pci")], srecs)
sv = kx.sriov([(b"10de", b"vfio-pci")], srecs, ssrs, sres["group_ids"], sres["group_off"], sres["group_members"])
ppf = np.where(np.arange(len(precs)) & 7, np.arange(len(precs)) & ~7, B.NO_PF).astype(np.uint32)
print("sriov withheld", int((sv["group_sriov"] != B.VIABLE).sum()), "pcie sriov nodes",
      len(kx.pcie_tree(precs, ppaths, poff, pmem, ppf)["key"]))
# mdev vGPUs on SR-IOV VFs: each mdev's PF joined against a PCI walk, and the slices with each vGPU's PF
mprecs, mpm, mps, mpwant = W.mdev_pf_walk(20480, 640, 20000)
assert np.array_equal(kx.mdev_pf(mprecs, mpm, mps), mpwant)
mpdevs = np.zeros(300, B.DRAMDEVPF_DTYPE)
mpdevs["dev"] = W.dra_mdev_devices(300)
mpdevs["physfn"][::2], mpdevs["physfn_device"][::2] = b"0000:41:00.0", b"2330"
print("mdev_pf resolved", int((mpwant != B.NO_PF).sum()), "slice bytes",
      len(kx.dra_slices_mdev_pf("d", "p", "n", 1, mpdevs, [("d/k", "", "NoSchedule")], np.full((300, 1), 5, np.int64))[0]))
# passthrough SR-IOV VFs: the slices with each VF's PF, untainted and with a one-entry table
pfdevs = W.dra_pf_devices(300)
print("dra_pf slice bytes", len(kx.dra_slices_pf("d", "p", "n", 1, pfdevs, [], None)[0]),
      len(kx.dra_slices_pf("d", "p", "n", 1, pfdevs, [("d/k", "", "NoSchedule")], np.full((300, 1), 5, np.int64))[0]))
# PCIe root ports and switches: the ports of a walk, then the slices untainted and with a one-entry table
prr, prp, pro, prm = W.pcie_ports_walk(3000)
prt, pst = kx.pcie_ports(prr, prp, pro, prm)
pcdevs = W.dra_pcie_devices(300)
print("pcie_ports switches", int((pst != B.PCIE_NO_KEY).sum()), "dra_pcie slice bytes",
      len(kx.dra_slices_pcie("d", "p", "n", 1, "pcie.example.com", pcdevs, [], None)[0]),
      len(kx.dra_slices_pcie("d", "p", "n", 1, "pcie.example.com", pcdevs, [("d/k", "", "NoSchedule")],
                             np.full((300, 1), 5, np.int64))[0]))
# the PCIe ports above every record (AER health): a PCI walk of switch trees with every chain end, then an mdev walk
apr, app = W.aer_port_walk(3000, depth=3, fanout=4, mixed=True)
apo, apf, apk = kx.aer_ports(apr, app)
amr, amp, _, _ = W.pcie_ports_mdev_walk(3000)
amo, amf, amk = kx.aer_ports(amr, amp)
print("aer_ports positions", int(apo[-1]), "ports", len(apk), "aer_ports_mdev positions", int(amo[-1]), "ports", len(amk))
# PCIe root ports and switches of vGPUs: the ports of an mdev walk, then both vGPU layouts untainted and with one taint
vmr, vmp, vmo, vmm = W.pcie_ports_mdev_walk(3000)
vrt, vst = kx.pcie_ports_mdev(vmr, vmp, vmo, vmm)
vmdevs, vfdevs = W.dra_mdev_pcie_devices(300), W.dra_vf_vgpu_pcie_devices(300)
print("pcie_ports_mdev switches", int((vst != B.PCIE_NO_KEY).sum()), "dra vgpu pcie slice bytes",
      len(kx.dra_slices_mdev_pcie("d", "p", "n", 1, "pcie.example.com", vmdevs, [], None)[0]),
      len(kx.dra_slices_mdev_pcie("d", "p", "n", 1, "pcie.example.com", vmdevs, [("d/k", "", "NoSchedule")],
                                  np.full((300, 1), 5, np.int64))[0]),
      len(kx.dra_slices_vf_vgpu_pcie("d", "p", "n", 1, "pcie.example.com", vfdevs, [], None)[0]),
      len(kx.dra_slices_vf_vgpu_pcie("d", "p", "n", 1, "pcie.example.com", vfdevs, [("d/k", "", "NoSchedule")],
                                     np.full((300, 1), 5, np.int64))[0]))
# resets between tenants: every member's function reset or bus-reset set, on the classify CSR
rrecs, rpaths, rrrs = W.reset_walk(20000)
rres = kx.classify_rules([(b"10de", b"vfio-pci")], rrecs)
rv = kx.reset_check([(b"10de", b"vfio-pci")], rrecs, rpaths, rrrs, B.RM_ALL, rres["group_off"], rres["group_members"])
print("reset withheld", int((rv["group_reset"] != B.VIABLE).sum()))
# Prometheus metrics: the size pass, the scan and the write pass over devices with reasons and AER values
mdevs, mstr, mrs = W.metrics_devices(20000)
print("metrics bytes", len(kx.metrics_devices(mdevs, mstr, mrs)))
# vGPUs on VFs: the type join and the per-type classify, with and without blockers
vrecs_, vvts, vtables = W.vf_vgpu_walk(20000)
vt = kx.vf_vgpu_types(vvts, vtables)
for viable in (False, True):
    vc = kx.classify_vf_vgpu([(b"10de", b"nvidia")], 1, vrecs_, vt["keys"], topo=viable, viable=viable)
    print("vf vgpu named", int((vt["status"] == B.VT_NAMED).sum()), "groups", vc["n_groups"], "types", vc["n_devids"])
# configured resource names: "*" on the passthrough rule beside the vGPU rule, with and without blockers
for viable in (False, True):
    nc = kx.classify_named([(b"10de", b"vfio-pci"), (b"10de", b"nvidia")], 2, vrecs_, vt["keys"], [(0, b"*", 0)],
                           topo=viable, viable=viable)
    print("named entries", nc["n_devids"], "slotted", int((nc["dev_slot"] != B.NO_SLOT).sum()))
# DRA ResourceSlices: one pool of 24 slices (the last one partial), and the empty pool
for dn_ in (3000, 0):
    blob, soff = kx.dra_slices("vfio.nvidia.com", "node-a", "node-a", 1, W.dra_devices(dn_))
    print("dra slices", len(soff) - 1, "bytes", len(blob))
# the vGPU layout of the same kernel: 24 slices and the empty pool
for dn_ in (3000, 0):
    blob, soff = kx.dra_slices_mdev("vgpu.nvidia.com", "node-a", "node-a", 1, W.dra_mdev_devices(dn_))
    print("dra mdev slices", len(soff) - 1, "bytes", len(blob))
# PCIe AER health: files shared by four vGPUs each at odd offsets; the taint list emitter with one and three entries,
# both layouts
ar = W.aer_records(20000, vgpus_per_parent=4)
_, gaer = kx.aer_health(ar["text"], ar["file_off"], ar["file_len"], 0, 0, ar["group_off"], ar["group_members"])
print("aer groups", len(gaer), "flagged", int(((gaer & 3) != 0).sum()))
tab3 = [("vfio.nvidia.com/unhealthy", "vfio-device-missing", "NoSchedule"),
        ("vfio.nvidia.com/pcie-aer", "fatal", "NoSchedule"), ("vfio.nvidia.com/pcie-aer", "nonfatal", "NoSchedule")]
since3 = np.full((3000, 3), -1, np.int64)
since3[::7, 0], since3[::5, 1], since3[1::5, 2] = 1767225600, 1767225660, 1767225720
blob, soff = kx.dra_slices_taints("vfio.nvidia.com", "node-a", "node-a", 1, W.dra_devices(3000), tab3[:1], since3[:, :1])
print("dra taints slices, one entry", len(soff) - 1, "bytes", len(blob))
blob, soff = kx.dra_slices_taints("vfio.nvidia.com", "node-a", "node-a", 1, W.dra_devices(3000), tab3, since3)
print("dra taints slices", len(soff) - 1, "bytes", len(blob))
blob, soff = kx.dra_slices_mdev_taints("vgpu.nvidia.com", "node-a", "node-a", 1, W.dra_mdev_devices(3000), tab3[:1],
                                       since3[:, :1])
print("dra mdev taints slices, one entry", len(soff) - 1, "bytes", len(blob))
blob, soff = kx.dra_slices_mdev_taints("vgpu.nvidia.com", "node-a", "node-a", 1, W.dra_mdev_devices(3000), tab3, since3)
print("dra mdev taints slices", len(soff) - 1, "bytes", len(blob))
# the VF-vGPU layout: untainted (24 slices and the empty pool) and with one and three taint entries
for dn_ in (3000, 0):
    blob, soff = kx.dra_slices_vf_vgpu("vgpu-vf.nvidia.com", "node-a", "node-a", 1, W.dra_vf_vgpu_devices(dn_), tab3, None)
    print("dra vf vgpu slices", len(soff) - 1, "bytes", len(blob))
blob, soff = kx.dra_slices_vf_vgpu("vgpu-vf.nvidia.com", "node-a", "node-a", 1, W.dra_vf_vgpu_devices(3000), tab3[:1],
                                   since3[:, :1])
print("dra vf vgpu taints slices, one entry", len(soff) - 1, "bytes", len(blob))
blob, soff = kx.dra_slices_vf_vgpu("vgpu-vf.nvidia.com", "node-a", "node-a", 1, W.dra_vf_vgpu_devices(3000), tab3, since3)
print("dra vf vgpu taints slices", len(soff) - 1, "bytes", len(blob))


# look-back state across epoch wraps (tests/test_gpu_lookback_state.py at reduced sizes): every user of the status
# words with at least two tiles, on a context whose epoch wraps every two epochs, against the default context
def lookback_pass(k, t):
    xr, mr = W.xpu_records(keys, n=4097, seed=7), W.mdev_records(n=4112, seed=7)
    dn = W.topo_dev_numa(2 * 4096 + 1)
    big = W.topo_requests(dn, n_req=3, avail=len(dn), size=700, must_max=3, seed=7)
    small = W.topo_requests(dn, n_req=4, avail=100, size=10, seed=8)
    prev, cur, ni = W.reconcile_pair(7, 1500)
    return [k.classify(W.cfg3_records(keys, n=70000, seed=7)), k.classify_rules(W.XPU_RULES, xr),
            k.classify_mdev(W.MDEV_RULES, mr), k.classify_topo(W.MDEV_RULES, W.topo_mdev_records(n=4112), mdev=True),
            k.names_blob(t, k.table_export(t)[2][:5000]), k.alloc_names(np.arange(5000, dtype=np.uint64), "amd.com/gpu"),
            k.mdev_names(mr, np.arange(4100, dtype=np.uint32)), k.lw_encode_topo(xr["iommu_group"], None, np.ones(4097, np.uint64)),
            k.cdi_emit(0, W.cfg5_devices(300), "amd.com/gpu"), k.cdi_emit_mdev(1, W.mdev_devices(300), "nvidia.com/vgpu"),
            k.reconcile(prev, cur, ni), k.preferred_allocation(dn, big[:1] + small + big[1:])]


def equal(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(equal(a[x], b[x]) for x in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(equal(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b)
    return a == b


os.environ["KXPU_SCAN_EPOCH_LIMIT"] = "3"
kw = K.Kxpu(0)
del os.environ["KXPU_SCAN_EPOCH_LIMIT"]
tw = kw.pciids_load(text * copies)
diff = [i for i, (a, b) in enumerate(zip(lookback_pass(kw, tw), lookback_pass(kx, tab))) if not equal(a, b)]
assert not diff, "calls %s differ across epoch wraps" % diff
print("look-back pass across epoch wraps: equal")
tw.free()
kw.close()
tab.free()
# full pci.ids model: build, export and lookup of every kind on the real file behind a block with the all-ones
# subsystem key (ffff ffff under device ffff of vendor ffff); the length is not a multiple of the 2 KiB chunk
ftext = b"ffff  Illegal\n\tffff  all\n\t\tffff ffff  ones\n\t\tffff fffe  x\n\t\t0000 0000  z\n" + text
assert len(ftext) % 2048
d_f = kx.dev_alloc(len(ftext)); kx.upload(d_f, np.frombuffer(ftext, np.uint8))
t_f = kx.pciids_load_device(d_f, len(ftext))
full = kx.full_load_device(d_f, len(ftext), t_f)
for kind in (0, 1, 2):
    fk, fo = kx.full_export(full, kind)
    fl = kx.full_lookup(full, kind, np.concatenate([fk, fk ^ np.uint64(32), np.array([(1 << 64) - 1], np.uint64)]))
    print("full kind", kind, "rows", len(fk), "hits", int((fl >= 0).sum()))
kx.full_free(full); t_f.free(); kx.dev_free(d_f)
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
bufs = []
# the same group at the peer slab's edges (tests/test_gpu_sharded.py): rank 1 with exactly 65 536 winner rows, rank 2
# with exactly 2 MiB of names, every offset past 2^32; parts of one length (comment lines behind the vendor line) so
# that the cuts fall between them
rng = np.random.default_rng(1)
alnum = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789", np.uint8)
parts = []
for v, n_dev, name_len in ((0x1000, 1, 8), (0x1001, 65536, 1), (0x1002, 32768, 64)):
    nm = alnum[rng.integers(0, len(alnum), n_dev * name_len)].tobytes()
    parts.append([b"%04x  V\n" % v, b"".join(b"\t%04x  " % d + nm[d * name_len:(d + 1) * name_len] + b"\n" for d in range(n_dev))])
plen = max(len(h) + len(b) for h, b in parts) + 2
edge = b""
for h, b in parts:
    pad = plen - len(h) - len(b)
    edge += h + b"".join(b"#" + b"p" * 998 + b"\n" for _ in range((pad - 2) // 1000)) + b"#" + b"p" * ((pad - 2) % 1000) + b"\n" + b
assert K.plan_shards(edge, 3) == [(0, plen), (plen, 2 * plen), (2 * plen, 3 * plen)]
shift = (1 << 32) - 1000
qe = np.concatenate([q, np.array([0x10010000, 0x1002ffff], np.uint32)])  # 770 keys: slices of 256, 256 and 258
shards = []
for r, (a, b) in enumerate(K.plan_shards(edge, 3)):
    k2 = m.ctxs[r]
    lo, hi = 256 * r, (770 if r == 2 else 256 * r + 256)
    d = k2.dev_alloc(b - a); k2.upload(d, np.frombuffer(edge[a:b], np.uint8))
    dq, dr = k2.dev_alloc((hi - lo) * 4), k2.dev_alloc(770 * 4)
    k2.upload(dq, qe[lo:hi])
    shards.append(dict(d_text=d, n=b - a, global_base=a + shift, d_keys=dq, nq=hi - lo, key_offset=lo, d_rows_all=dr))
    bufs.append((k2, d, dq, dr))
tabs = m.pciids_join(shards, 770)
_, eoffs, erows = m.ctxs[1].table_export(tabs[1])
got = m.ctxs[1].download(shards[1]["d_rows_all"], 770 * 4, np.int32)
names = m.ctxs[2].names_blob(tabs[2], erows)[0]
assert [t.rows for t in tabs] == [1 + 65536 + 32768] * 3 and int(eoffs.min()) >= shift and got[768] >= 0 and got[769] == -1
assert len(names) == 8 + 65536 + (2 << 20)
print("sharded slab edges rows", tabs[0].rows, "name bytes", len(names))
for t in tabs:
    t.free()
for k2, d, dq, dr in bufs:
    k2.dev_free(d); k2.dev_free(dq); k2.dev_free(dr)
m.close()
