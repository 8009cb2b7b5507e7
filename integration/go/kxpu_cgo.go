// kxpu_cgo.go -- the cgo shim of INTEGRATION.md as a file: drop it into pkg/device_plugin of the
// reference next to device_plugin.go (build tag keeps the stock CPU path selectable).
// NOT compiled in this repository: the build image has no Go toolchain.
//go:build kxpu

package device_plugin

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../lib -lkxpu
#include <stdlib.h>
#include "kxpu.h"
*/
import "C"

import (
	"fmt"
	"os"
	"runtime"
	"strings"
	"unsafe"

	pluginapi "k8s.io/kubelet/pkg/apis/deviceplugin/v1beta1"
)

type kxpu struct {
	ctx   *C.kxpu_ctx
	table *C.kxpu_table // parsed pci.ids, built once
}

func kxCheck(ctx *C.kxpu_ctx, what string, rc C.int32_t) error {
	if rc == C.KXPU_OK {
		return nil
	}
	return fmt.Errorf("%s: %s (%s)", what, C.GoString(C.kxpu_strerror(rc)), C.GoString(C.kxpu_last_error(ctx)))
}

// The library has no CPU path: without a GPU on the NVIDIA driver kxpu_ctx_create returns
// KXPU_E_NOGPU.  A node whose GPUs are ALL bound to vfio-pci (the reference's normal deployment)
// therefore cannot use it; InitiateDevicePlugin calls newKxpu once and, on error, logs it and keeps
// the stock functions (createIommuDeviceMap, getDeviceName, generateCDISpec are untouched in the
// tree and selected by `if kx == nil`).  That is the host's choice between two implementations,
// not a fallback inside the library; after a successful create every kxpu_* error is fatal.
func newKxpu(ordinal int) (*kxpu, error) {
	k := &kxpu{}
	if rc := C.kxpu_ctx_create(C.int32_t(ordinal), &k.ctx); rc != C.KXPU_OK {
		return nil, fmt.Errorf("kxpu_ctx_create: %s", C.GoString(C.kxpu_strerror(rc)))
	}
	return k, nil
}

// S2: parse pciIdsFilePath once (replaces the per-id rescan of getDeviceName/locateVendor).
func (k *kxpu) loadPciIds(path string) error {
	text, err := os.ReadFile(path)
	if err != nil {
		return err
	}
	var p *C.uint8_t
	if len(text) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&text[0])) // borrowed for the call only
	}
	return kxCheck(k.ctx, "kxpu_pciids_load", C.kxpu_pciids_load(k.ctx, p, C.size_t(len(text)), &k.table))
}

// S2: batched getDeviceName for NVIDIA device ids ("" = not found, like the reference).
func (k *kxpu) deviceNames(ids []string) ([]string, error) {
	keys := make([]C.uint32_t, len(ids))
	for i, id := range ids {
		var d uint32
		if _, err := fmt.Sscanf(id, "%04x", &d); err != nil || len(id) != 4 {
			keys[i] = 0xffffffff // never present under 10de -> ""
			continue
		}
		keys[i] = C.uint32_t(0x10de<<16 | d)
	}
	rows := make([]C.int32_t, len(ids))
	offs := make([]C.uint32_t, len(ids)+1)
	if len(ids) == 0 {
		return nil, nil
	}
	if err := kxCheck(k.ctx, "kxpu_lookup", C.kxpu_lookup(k.ctx, k.table, &keys[0], C.size_t(len(ids)), &rows[0])); err != nil {
		return nil, err
	}
	var need C.size_t
	C.kxpu_names(k.ctx, k.table, &rows[0], C.size_t(len(ids)), nil, 0, &offs[0], &need) // sizing call
	buf := make([]byte, need+1)
	if err := kxCheck(k.ctx, "kxpu_names", C.kxpu_names(k.ctx, k.table, &rows[0], C.size_t(len(ids)),
		(*C.uint8_t)(unsafe.Pointer(&buf[0])), need, &offs[0], &need)); err != nil {
		return nil, err
	}
	out := make([]string, len(ids))
	for i := range ids {
		out[i] = string(buf[offs[i]:offs[i+1]])
	}
	return out, nil
}

// S1/S4: classify the raw sysfs records gathered by the walk.
// kxpu_classify_out is a struct of seven output pointers.  `out` itself lives in Go memory, so cgo
// (cgocheck=1, the default) inspects it and refuses Go pointers to UNPINNED Go memory inside it
// ("cgo argument has Go pointer to unpinned Go pointer").  runtime.Pinner (Go 1.21+) pins the seven
// backing arrays for the duration of the call; the library keeps none of them (include/kxpu.h).
func (k *kxpu) classify(recs []C.kxpu_devrec) (accept, gids, goff, gmem []uint32, dids []uint64, doff, dgrp []uint32, err error) {
	n := len(recs)
	accept, gids, goff, gmem = make([]uint32, n), make([]uint32, n), make([]uint32, n+1), make([]uint32, n)
	dids, doff, dgrp = make([]uint64, n), make([]uint32, n+1), make([]uint32, n)
	if n == 0 {
		return
	}
	var pin runtime.Pinner
	defer pin.Unpin()
	pin.Pin(&accept[0])
	pin.Pin(&gids[0])
	pin.Pin(&goff[0])
	pin.Pin(&gmem[0])
	pin.Pin(&dids[0])
	pin.Pin(&doff[0])
	pin.Pin(&dgrp[0])
	var out C.kxpu_classify_out
	out.accept_index = (*C.uint32_t)(unsafe.Pointer(&accept[0]))
	out.group_ids = (*C.uint32_t)(unsafe.Pointer(&gids[0]))
	out.group_off = (*C.uint32_t)(unsafe.Pointer(&goff[0]))
	out.group_members = (*C.uint32_t)(unsafe.Pointer(&gmem[0]))
	out.dev_ids = (*C.uint64_t)(unsafe.Pointer(&dids[0]))
	out.dev_off = (*C.uint32_t)(unsafe.Pointer(&doff[0]))
	out.dev_groups = (*C.uint32_t)(unsafe.Pointer(&dgrp[0]))
	err = kxCheck(k.ctx, "kxpu_classify", C.kxpu_classify(k.ctx, &recs[0], C.size_t(n), &out))
	gids, goff, gmem = gids[:out.n_groups], goff[:out.n_groups+1], gmem[:out.n_accepted]
	dids, doff, dgrp = dids[:out.n_devids], doff[:out.n_devids+1], dgrp[:out.n_groups]
	return
}

// S2, start-up form: pci.ids text + every device id of deviceMap in ONE call and one host round trip
// (kxpu_pciids_join: for the 1.4 MB file one cooperative kernel parses, folds, names and joins).
func (k *kxpu) loadAndJoin(path string, keys []uint32) ([]int32, error) {
	text, err := os.ReadFile(path)
	if err != nil {
		return nil, err
	}
	rows := make([]int32, len(keys))
	var tp *C.uint8_t
	var kp *C.uint32_t
	var rp *C.int32_t
	if len(text) > 0 {
		tp = (*C.uint8_t)(unsafe.Pointer(&text[0]))
	}
	if len(keys) > 0 {
		kp = (*C.uint32_t)(unsafe.Pointer(&keys[0]))
		rp = (*C.int32_t)(unsafe.Pointer(&rows[0]))
	}
	err = kxCheck(k.ctx, "kxpu_pciids_join", C.kxpu_pciids_join(k.ctx, tp, C.size_t(len(text)), kp, C.size_t(len(keys)), rp, &k.table))
	return rows, err
}

// S3: CDI document bytes (format 0 = YAML as the reference's live path, 1 = JSON).
func (k *kxpu) cdiEmit(format int, devs []C.kxpu_cdidev) ([]byte, error) {
	var p *C.kxpu_cdidev
	if len(devs) > 0 {
		p = &devs[0]
	}
	var n C.size_t
	C.kxpu_cdi_emit(k.ctx, C.int32_t(format), p, C.size_t(len(devs)), nil, 0, &n) // sizing call
	buf := make([]byte, n+1)
	err := kxCheck(k.ctx, "kxpu_cdi_emit", C.kxpu_cdi_emit(k.ctx, C.int32_t(format), p, C.size_t(len(devs)),
		(*C.uint8_t)(unsafe.Pointer(&buf[0])), n, &n))
	return buf[:n], err
}

// S5: CDI device names of an Allocate response.
func (k *kxpu) allocNames(idx []uint64) ([]string, error) {
	if len(idx) == 0 {
		return nil, nil
	}
	offs := make([]C.uint32_t, len(idx)+1)
	buf := make([]byte, 36*len(idx))
	var need C.size_t
	err := kxCheck(k.ctx, "kxpu_alloc_names", C.kxpu_alloc_names(k.ctx, (*C.uint64_t)(unsafe.Pointer(&idx[0])), C.size_t(len(idx)),
		(*C.uint8_t)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)), &offs[0], &need))
	out := make([]string, len(idx))
	for i := range idx {
		out[i] = string(buf[offs[i]:offs[i+1]])
	}
	return out, err
}

// ---- accelerators of any configured vendor (README TODO "To support other GPUs")

// xpuClass is one accelerator class the plugin serves: the constants nvidiaVendorID (device_plugin.go:19),
// "vfio-pci" (:156), DevicePluginNamespace / CdiVendorClass (generic_device_plugin.go:26,31) and the CDI file
// stem (device_plugin.go:79) become fields.  The default list is {"10de", "vfio-pci", "nvidia.com",
// "nvidia.com/gpu", "cdi-vfio-xxxx"}.
type xpuClass struct {
	Vendor, Driver, Namespace, Kind, FileStem string
	// device id ("2330") or "*" -> resource name (kxpu_classify_named); nil: named by pci.ids, one resource per id
	ResourceNames map[string]string
}

// S1 with a class list: one rule per class (rule index == class index).  devRule[d] is the class of deviceMap
// entry d; the same device id can appear under two classes.
func (k *kxpu) classifyRules(classes []xpuClass, recs []C.kxpu_devrec) (accept, gids, goff, gmem []uint32, dids []uint64,
	doff, dgrp []uint32, devRule []uint8, err error) {
	n := len(recs)
	accept, gids, goff, gmem = make([]uint32, n), make([]uint32, n), make([]uint32, n+1), make([]uint32, n)
	dids, doff, dgrp, devRule = make([]uint64, n), make([]uint32, n+1), make([]uint32, n), make([]uint8, n)
	if n == 0 {
		return
	}
	rules := make([]C.kxpu_xpu_rule, len(classes))
	for i, c := range classes {
		for j := 0; j < len(c.Vendor) && j < len(rules[i].vendor); j++ {
			rules[i].vendor[j] = C.char(c.Vendor[j])
		}
		for j := 0; j < len(c.Driver) && j < len(rules[i].driver); j++ {
			rules[i].driver[j] = C.char(c.Driver[j])
		}
	}
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, p := range []*uint32{&accept[0], &gids[0], &goff[0], &gmem[0], &doff[0], &dgrp[0]} {
		pin.Pin(p)
	}
	pin.Pin(&dids[0])
	var out C.kxpu_classify_out
	out.accept_index = (*C.uint32_t)(unsafe.Pointer(&accept[0]))
	out.group_ids = (*C.uint32_t)(unsafe.Pointer(&gids[0]))
	out.group_off = (*C.uint32_t)(unsafe.Pointer(&goff[0]))
	out.group_members = (*C.uint32_t)(unsafe.Pointer(&gmem[0]))
	out.dev_ids = (*C.uint64_t)(unsafe.Pointer(&dids[0]))
	out.dev_off = (*C.uint32_t)(unsafe.Pointer(&doff[0]))
	out.dev_groups = (*C.uint32_t)(unsafe.Pointer(&dgrp[0]))
	var rp *C.kxpu_xpu_rule
	if len(rules) > 0 {
		rp = &rules[0]
	}
	err = kxCheck(k.ctx, "kxpu_classify_rules", C.kxpu_classify_rules(k.ctx, rp, C.size_t(len(rules)), &recs[0], C.size_t(n), &out,
		(*C.uint8_t)(unsafe.Pointer(&devRule[0]))))
	gids, goff, gmem = gids[:out.n_groups], goff[:out.n_groups+1], gmem[:out.n_accepted]
	dids, doff, dgrp, devRule = dids[:out.n_devids], doff[:out.n_devids+1], dgrp[:out.n_groups], devRule[:out.n_devids]
	return
}

// S3 for one class: the CDI document of that class's devices with its kind.
func (k *kxpu) cdiEmitKind(format int, kind string, devs []C.kxpu_cdidev) ([]byte, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	var p *C.kxpu_cdidev
	if len(devs) > 0 {
		p = &devs[0]
	}
	var n C.size_t
	C.kxpu_cdi_emit_kind(k.ctx, C.int32_t(format), ck, p, C.size_t(len(devs)), nil, 0, &n) // sizing call
	buf := make([]byte, n+1)
	err := kxCheck(k.ctx, "kxpu_cdi_emit_kind", C.kxpu_cdi_emit_kind(k.ctx, C.int32_t(format), ck, p, C.size_t(len(devs)),
		(*C.uint8_t)(unsafe.Pointer(&buf[0])), n, &n))
	return buf[:n], err
}

// S5 for one class: "<kind>=<index>" names of an Allocate response.
func (k *kxpu) allocNamesKind(kind string, idx []uint64) ([]string, error) {
	if len(idx) == 0 {
		return nil, nil
	}
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	offs := make([]C.uint32_t, len(idx)+1)
	buf := make([]byte, (len(kind)+22)*len(idx))
	var need C.size_t
	err := kxCheck(k.ctx, "kxpu_alloc_names_kind", C.kxpu_alloc_names_kind(k.ctx, ck, (*C.uint64_t)(unsafe.Pointer(&idx[0])),
		C.size_t(len(idx)), (*C.uint8_t)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)), &offs[0], &need))
	out := make([]string, len(idx))
	for i := range idx {
		out[i] = string(buf[offs[i]:offs[i+1]])
	}
	return out, err
}

// vGPUs (mediated devices): a vGPU class is an xpuClass whose Vendor is the parent PCI device's vendor and whose
// Driver is the mdev's driver.  The walk of /sys/bus/mdev/devices fills one C.kxpu_mdevrec per entry.

// S1 for the mdev walk: classifyRules' outputs, except that dids[d] is the index of the first record carrying
// entry d's type key; typeKeys returns the keys themselves.
func (k *kxpu) classifyMdev(classes []xpuClass, recs []C.kxpu_mdevrec) (accept, gids, goff, gmem []uint32, dids []uint64,
	doff, dgrp []uint32, devRule []uint8, err error) {
	n := len(recs)
	accept, gids, goff, gmem = make([]uint32, n), make([]uint32, n), make([]uint32, n+1), make([]uint32, n)
	dids, doff, dgrp, devRule = make([]uint64, n), make([]uint32, n+1), make([]uint32, n), make([]uint8, n)
	if n == 0 {
		return
	}
	rules := make([]C.kxpu_xpu_rule, len(classes))
	for i, c := range classes {
		for j := 0; j < len(c.Vendor) && j < len(rules[i].vendor); j++ {
			rules[i].vendor[j] = C.char(c.Vendor[j])
		}
		for j := 0; j < len(c.Driver) && j < len(rules[i].driver); j++ {
			rules[i].driver[j] = C.char(c.Driver[j])
		}
	}
	var pin runtime.Pinner
	defer pin.Unpin()
	for _, p := range []*uint32{&accept[0], &gids[0], &goff[0], &gmem[0], &doff[0], &dgrp[0]} {
		pin.Pin(p)
	}
	pin.Pin(&dids[0])
	var out C.kxpu_classify_out
	out.accept_index = (*C.uint32_t)(unsafe.Pointer(&accept[0]))
	out.group_ids = (*C.uint32_t)(unsafe.Pointer(&gids[0]))
	out.group_off = (*C.uint32_t)(unsafe.Pointer(&goff[0]))
	out.group_members = (*C.uint32_t)(unsafe.Pointer(&gmem[0]))
	out.dev_ids = (*C.uint64_t)(unsafe.Pointer(&dids[0]))
	out.dev_off = (*C.uint32_t)(unsafe.Pointer(&doff[0]))
	out.dev_groups = (*C.uint32_t)(unsafe.Pointer(&dgrp[0]))
	var rp *C.kxpu_xpu_rule
	if len(rules) > 0 {
		rp = &rules[0]
	}
	err = kxCheck(k.ctx, "kxpu_classify_mdev", C.kxpu_classify_mdev(k.ctx, rp, C.size_t(len(rules)), &recs[0], C.size_t(n), &out,
		(*C.uint8_t)(unsafe.Pointer(&devRule[0]))))
	gids, goff, gmem = gids[:out.n_groups], goff[:out.n_groups+1], gmem[:out.n_accepted]
	dids, doff, dgrp, devRule = dids[:out.n_devids], doff[:out.n_devids+1], dgrp[:out.n_groups], devRule[:out.n_devids]
	return
}

// The type keys (resource-name suffixes) of recs[idx[j]].
func (k *kxpu) typeKeys(recs []C.kxpu_mdevrec, idx []uint32) ([]string, error) {
	if len(idx) == 0 || len(recs) == 0 {
		return nil, nil
	}
	offs := make([]C.uint32_t, len(idx)+1)
	buf := make([]byte, 40*len(idx)+1)
	var need C.size_t
	err := kxCheck(k.ctx, "kxpu_mdev_names", C.kxpu_mdev_names(k.ctx, &recs[0], C.size_t(len(recs)),
		(*C.uint32_t)(unsafe.Pointer(&idx[0])), C.size_t(len(idx)), (*C.uint8_t)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)),
		&offs[0], &need))
	out := make([]string, len(idx))
	for j := range idx {
		out[j] = string(buf[offs[j]:offs[j+1]])
	}
	return out, err
}

// S3 for one vGPU class: the CDI document with the mdev annotation per device.
func (k *kxpu) cdiEmitMdev(format int, kind string, devs []C.kxpu_mdevcdi) ([]byte, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	var p *C.kxpu_mdevcdi
	if len(devs) > 0 {
		p = &devs[0]
	}
	var n C.size_t
	C.kxpu_cdi_emit_mdev(k.ctx, C.int32_t(format), ck, p, C.size_t(len(devs)), nil, 0, &n) // sizing call
	buf := make([]byte, n+1)
	err := kxCheck(k.ctx, "kxpu_cdi_emit_mdev", C.kxpu_cdi_emit_mdev(k.ctx, C.int32_t(format), ck, p, C.size_t(len(devs)),
		(*C.uint8_t)(unsafe.Pointer(&buf[0])), n, &n))
	return buf[:n], err
}

// NUMA topology (ABI v5).  With topology on, the walks fill numa_node / KXPU_REC_NUMA from <entry>/numa_node (an mdev:
// <uuid>/../numa_node), classify returns one NUMA mask per group, and the Go call sites use the masks:
//   - createDevicePlugins: pluginapi.Device{ID, Health, Topology: topologyInfo(mask)} for every group;
//   - Register: pluginapi.DevicePluginOptions{GetPreferredAllocationAvailable: true};
//   - GetDevicePluginOptions returns the same options; GetPreferredAllocation calls preferredAllocation once per
//     PreferredAllocationRequest with the positions of the request's IDs in dpi.devs.

// classifyRules / classifyMdev plus the NUMA mask of every group (mdev selects kxpu_classify_mdev_topo; recs is then a
// []C.kxpu_mdevrec passed as its first element's address and n).
func (k *kxpu) groupNuma(out *C.kxpu_classify_out, rules []C.kxpu_xpu_rule, recs unsafe.Pointer, n int, mdev bool,
	devRule []uint8) ([]uint64, error) {
	gnuma := make([]uint64, n)
	if n == 0 {
		return gnuma, nil
	}
	var rp *C.kxpu_xpu_rule
	if len(rules) > 0 {
		rp = &rules[0]
	}
	var rc C.int32_t
	if mdev {
		rc = C.kxpu_classify_mdev_topo(k.ctx, rp, C.size_t(len(rules)), (*C.kxpu_mdevrec)(recs), C.size_t(n), out,
			(*C.uint8_t)(unsafe.Pointer(&devRule[0])), (*C.uint64_t)(unsafe.Pointer(&gnuma[0])))
	} else {
		rc = C.kxpu_classify_topo(k.ctx, rp, C.size_t(len(rules)), (*C.kxpu_devrec)(recs), C.size_t(n), out,
			(*C.uint8_t)(unsafe.Pointer(&devRule[0])), (*C.uint64_t)(unsafe.Pointer(&gnuma[0])))
	}
	return gnuma[:out.n_groups], kxCheck(k.ctx, "kxpu_classify_topo", rc)
}

// IOMMU group viability (ABI v8).  With it on, the PCI walk sets KXPU_REC_BLOCKS, the group and the driver on every
// function that is not a class candidate and is bound to a driver outside the viability list, and the Go call sites use
// the first blocker of each group:
//   - createIommuDeviceMap: classifyViable in place of classifyRules / groupNuma, one "<bdf> is bound to <driver>" per
//     group with a blocker;
//   - createDevicePlugins / ListAndWatch: such a group's Device is sent Unhealthy whatever its health watch says;
//   - Allocate: a request naming such a group fails before any read.

// classifyRules plus the first blocking record of every group (KXPU_VIABLE: none); topo also fills the NUMA masks
// (kxpu_classify_topo's), else gnuma is nil.  out must be wired and pinned as for classifyRules.
func (k *kxpu) classifyViable(out *C.kxpu_classify_out, rules []C.kxpu_xpu_rule, recs []C.kxpu_devrec, devRule []uint8,
	topo bool) (blockers []uint32, gnuma []uint64, err error) {
	n := len(recs)
	blockers = make([]uint32, n)
	if topo {
		gnuma = make([]uint64, n)
	}
	if n == 0 {
		return blockers, gnuma, nil
	}
	var rp *C.kxpu_xpu_rule
	if len(rules) > 0 {
		rp = &rules[0]
	}
	var np *C.uint64_t
	if topo {
		np = (*C.uint64_t)(unsafe.Pointer(&gnuma[0]))
	}
	rc := C.kxpu_classify_viable(k.ctx, rp, C.size_t(len(rules)), &recs[0], C.size_t(n), out,
		(*C.uint8_t)(unsafe.Pointer(&devRule[0])), np, (*C.uint32_t)(unsafe.Pointer(&blockers[0])))
	if topo {
		gnuma = gnuma[:out.n_groups]
	}
	return blockers[:out.n_groups], gnuma, kxCheck(k.ctx, "kxpu_classify_viable", rc)
}

// pluginapi.TopologyInfo of a mask: one NUMANode per set bit, ascending; nil for 0 (no topology)
func topologyInfo(mask uint64) *pluginapi.TopologyInfo {
	if mask == 0 {
		return nil
	}
	t := &pluginapi.TopologyInfo{}
	for n := 0; n < 64; n++ {
		if mask>>n&1 == 1 {
			t.Nodes = append(t.Nodes, &pluginapi.NUMANode{ID: int64(n)})
		}
	}
	return t
}

// ListAndWatchResponse bytes with Device.topology (what proto.Marshal of the response gives).
func (k *kxpu) lwEncodeTopo(groups []uint32, healthy []uint8, masks []uint64) ([]byte, error) {
	if len(groups) == 0 {
		return nil, nil
	}
	g, h, m := (*C.uint32_t)(unsafe.Pointer(&groups[0])), (*C.uint8_t)(unsafe.Pointer(&healthy[0])), (*C.uint64_t)(unsafe.Pointer(&masks[0]))
	var n C.size_t
	C.kxpu_lw_encode_topo(k.ctx, g, h, m, C.size_t(len(groups)), nil, 0, &n) // sizing call
	buf := make([]byte, n+1)
	err := kxCheck(k.ctx, "kxpu_lw_encode_topo", C.kxpu_lw_encode_topo(k.ctx, g, h, m, C.size_t(len(groups)),
		(*C.uint8_t)(unsafe.Pointer(&buf[0])), n, &n))
	return buf[:n], err
}

// GetPreferredAllocation for all container requests of one PreferredAllocationRequest: avail / must hold positions in
// dpi.devs, masks[d] is dpi.devs[d]'s NUMA mask.  Returns the positions of each request's answer.
func (k *kxpu) preferredAllocation(masks []uint64, avail, must [][]uint32, size []uint32) ([][]uint32, error) {
	nreq := len(size)
	aoff, moff := make([]uint32, nreq+1), make([]uint32, nreq+1)
	var a, m []uint32
	total := 0
	for q := 0; q < nreq; q++ {
		a, m = append(a, avail[q]...), append(m, must[q]...)
		aoff[q+1], moff[q+1] = uint32(len(a)), uint32(len(m))
		total += int(size[q])
	}
	a, m = append(a, 0), append(m, 0) // valid pointers for empty lists
	masks = append(masks, 0)
	sz := append(size, 0)
	out, ooff := make([]uint32, total+1), make([]uint32, nreq+1)
	err := kxCheck(k.ctx, "kxpu_preferred_allocation", C.kxpu_preferred_allocation(k.ctx,
		(*C.uint64_t)(unsafe.Pointer(&masks[0])), C.size_t(len(masks)-1), (*C.uint32_t)(unsafe.Pointer(&aoff[0])),
		(*C.uint32_t)(unsafe.Pointer(&a[0])), (*C.uint32_t)(unsafe.Pointer(&moff[0])), (*C.uint32_t)(unsafe.Pointer(&m[0])),
		(*C.uint32_t)(unsafe.Pointer(&sz[0])), C.size_t(nreq), (*C.uint32_t)(unsafe.Pointer(&out[0])),
		(*C.uint32_t)(unsafe.Pointer(&ooff[0]))))
	res := make([][]uint32, nreq)
	for q := 0; err == nil && q < nreq; q++ {
		res[q] = out[ooff[q]:ooff[q+1]]
	}
	return res, err
}

// PCIe topology (ABI v7).  With pcieTopology on, the PCI walk also runs os.Readlink(<basePath>/<entry>) per entry and
// keeps the target from its first component that begins with "pci" (pciPath); after classify, pcieTree builds the walk's
// forest, every passthrough pluginapi.Device keeps its group's node beside it, GetDevicePluginOptions reports
// GetPreferredAllocationAvailable, and GetPreferredAllocation of a passthrough plugin calls
// preferredAllocationPcie with the forest shared by all plugins of the walk (vGPU plugins keep preferredAllocation).

// the kxpu_pcipath of one link target: unknown (len 0) without a "pci" component or past 120 bytes
func pciPath(target string) C.kxpu_pcipath {
	var p C.kxpu_pcipath
	for at := 0; at < len(target); {
		if strings.HasPrefix(target[at:], "pci") {
			if rest := target[at:]; len(rest) <= len(p.path) {
				for i := 0; i < len(rest); i++ {
					p.path[i] = C.char(rest[i])
				}
				p.len = C.uint8_t(len(rest))
			}
			return p
		}
		slash := strings.IndexByte(target[at:], '/')
		if slash < 0 {
			break
		}
		at += slash + 1
	}
	return p
}

// the forest of a walk: recs / paths at the same indices, goff / gmem the classify CSR of nGroups groups
func (k *kxpu) pcieTree(recs []C.kxpu_devrec, paths []C.kxpu_pcipath, goff, gmem []uint32, nGroups int) (gnode, parent []uint32,
	depth []uint8, err error) {
	capN := 8*nGroups + 1
	gnode, parent, depth = make([]uint32, nGroups+1), make([]uint32, capN), make([]uint8, capN)
	key := make([]uint64, capN)
	var nn C.uint32_t
	var r unsafe.Pointer
	var pp *C.kxpu_pcipath
	if len(recs) > 0 {
		r, pp = unsafe.Pointer(&recs[0]), &paths[0]
	}
	gm := append(gmem, 0) // a valid pointer for an empty walk
	err = kxCheck(k.ctx, "kxpu_pcie_tree", C.kxpu_pcie_tree(k.ctx, (*C.kxpu_devrec)(r), pp, C.size_t(len(recs)),
		(*C.uint32_t)(unsafe.Pointer(&goff[0])), (*C.uint32_t)(unsafe.Pointer(&gm[0])), C.size_t(nGroups),
		(*C.uint32_t)(unsafe.Pointer(&gnode[0])), (*C.uint64_t)(unsafe.Pointer(&key[0])),
		(*C.uint32_t)(unsafe.Pointer(&parent[0])), (*C.uint8_t)(unsafe.Pointer(&depth[0])), &nn))
	return gnode[:nGroups], parent[:nn], depth[:nn], err
}

// the root port and nearest switch of each group (an addition to ABI v14, detected by symbol): pcieTree's inputs, one
// function key per group or C.KXPU_PCIE_NO_KEY in each output.  Called once per PCI walk when draPcieConfig.DraPcieDomain
// is set.
func (k *kxpu) pciePorts(recs []C.kxpu_devrec, paths []C.kxpu_pcipath, goff, gmem []uint32, nGroups int) (rootPort,
	pcieSwitch []uint64, err error) {
	rootPort, pcieSwitch = make([]uint64, nGroups+1), make([]uint64, nGroups+1)
	var r unsafe.Pointer
	var pp *C.kxpu_pcipath
	if len(recs) > 0 {
		r, pp = unsafe.Pointer(&recs[0]), &paths[0]
	}
	gm := append(gmem, 0) // a valid pointer for an empty walk
	err = kxCheck(k.ctx, "kxpu_pcie_ports", C.kxpu_pcie_ports(k.ctx, (*C.kxpu_devrec)(r), pp, C.size_t(len(recs)),
		(*C.uint32_t)(unsafe.Pointer(&goff[0])), (*C.uint32_t)(unsafe.Pointer(&gm[0])), C.size_t(nGroups),
		(*C.uint64_t)(unsafe.Pointer(&rootPort[0])), (*C.uint64_t)(unsafe.Pointer(&pcieSwitch[0]))))
	return rootPort[:nGroups], pcieSwitch[:nGroups], err
}

// the root port and nearest switch of each mdev group (an addition to ABI v14, detected by symbol): pcieTreeMdev's
// inputs, the keys of each group's parent GPU, or C.KXPU_PCIE_NO_KEY.  Called once per mdev walk when
// draVgpuPcieConfig.DraVgpuPcie is set and a vGPU class has a draDriver.
func (k *kxpu) pciePortsMdev(recs []C.kxpu_mdevrec, paths []C.kxpu_pcipath, goff, gmem []uint32, nGroups int) (rootPort,
	pcieSwitch []uint64, err error) {
	rootPort, pcieSwitch = make([]uint64, nGroups+1), make([]uint64, nGroups+1)
	var r unsafe.Pointer
	var pp *C.kxpu_pcipath
	if len(recs) > 0 {
		r, pp = unsafe.Pointer(&recs[0]), &paths[0]
	}
	gm := append(gmem, 0) // a valid pointer for an empty walk
	err = kxCheck(k.ctx, "kxpu_pcie_ports_mdev", C.kxpu_pcie_ports_mdev(k.ctx, (*C.kxpu_mdevrec)(r), pp,
		C.size_t(len(recs)), (*C.uint32_t)(unsafe.Pointer(&goff[0])), (*C.uint32_t)(unsafe.Pointer(&gm[0])),
		C.size_t(nGroups), (*C.uint64_t)(unsafe.Pointer(&rootPort[0])), (*C.uint64_t)(unsafe.Pointer(&pcieSwitch[0]))))
	return rootPort[:nGroups], pcieSwitch[:nGroups], err
}

// the PCIe ports above every record (an addition to ABI v14, detected by symbol): ports of record i are
// portOf[portOff[i]:portOff[i+1]], nearest first, and portKey[p] is port p's function key.  Called once per PCI walk
// when aerPortHealth is set; computeAer then reads each distinct port's aer_dev_* files after a group's own members.
func (k *kxpu) aerPorts(recs []C.kxpu_devrec, paths []C.kxpu_pcipath) (portOff, portOf []uint32, portKey []uint64, err error) {
	n := len(recs)
	portOff = make([]uint32, n+1)
	portOf, portKey = make([]uint32, C.KXPU_PCIE_MAX_DEPTH*n+1), make([]uint64, C.KXPU_PCIE_MAX_DEPTH*n+1)
	var r unsafe.Pointer
	var pp *C.kxpu_pcipath
	if n > 0 {
		r, pp = unsafe.Pointer(&recs[0]), &paths[0]
	}
	var nk C.uint32_t
	err = kxCheck(k.ctx, "kxpu_aer_ports", C.kxpu_aer_ports(k.ctx, (*C.kxpu_devrec)(r), pp, C.size_t(n),
		(*C.uint32_t)(unsafe.Pointer(&portOff[0])), (*C.uint32_t)(unsafe.Pointer(&portOf[0])),
		(*C.uint64_t)(unsafe.Pointer(&portKey[0])), &nk))
	return portOff, portOf[:portOff[n]], portKey[:nk], err
}

// aerPorts for the mdev walk: the ports above each mdev's parent GPU.  Called once per mdev walk when aerPortHealth is
// set.
func (k *kxpu) aerPortsMdev(recs []C.kxpu_mdevrec, paths []C.kxpu_pcipath) (portOff, portOf []uint32, portKey []uint64, err error) {
	n := len(recs)
	portOff = make([]uint32, n+1)
	portOf, portKey = make([]uint32, C.KXPU_PCIE_MAX_DEPTH*n+1), make([]uint64, C.KXPU_PCIE_MAX_DEPTH*n+1)
	var r unsafe.Pointer
	var pp *C.kxpu_pcipath
	if n > 0 {
		r, pp = unsafe.Pointer(&recs[0]), &paths[0]
	}
	var nk C.uint32_t
	err = kxCheck(k.ctx, "kxpu_aer_ports_mdev", C.kxpu_aer_ports_mdev(k.ctx, (*C.kxpu_mdevrec)(r), pp, C.size_t(n),
		(*C.uint32_t)(unsafe.Pointer(&portOff[0])), (*C.uint32_t)(unsafe.Pointer(&portOf[0])),
		(*C.uint64_t)(unsafe.Pointer(&portKey[0])), &nk))
	return portOff, portOf[:portOff[n]], portKey[:nk], err
}

// pcieTree over records that carry only their address, one per link target (walk order): what pcieTree sees of a walk
func (k *kxpu) pcieTreeOfLinks(bdfs, targets []string, goff, gmem []uint32) (gnode, parent []uint32, depth []uint8, err error) {
	recs, paths := make([]C.kxpu_devrec, len(bdfs)), make([]C.kxpu_pcipath, len(bdfs))
	for i, b := range bdfs {
		for j := 0; j < len(b) && j < len(recs[i].bdf)-1; j++ {
			recs[i].bdf[j] = C.char(b[j])
		}
		paths[i] = pciPath(targets[i])
	}
	return k.pcieTree(recs, paths, goff, gmem, len(goff)-1)
}

// preferredAllocation with each device's PCIe node (nodes[d] of dpi.devs[d]) and the walk's forest
func (k *kxpu) preferredAllocationPcie(masks []uint64, nodes, parent []uint32, depth []uint8, avail, must [][]uint32,
	size []uint32) ([][]uint32, error) {
	nreq := len(size)
	aoff, moff := make([]uint32, nreq+1), make([]uint32, nreq+1)
	var a, m []uint32
	total := 0
	for q := 0; q < nreq; q++ {
		a, m = append(a, avail[q]...), append(m, must[q]...)
		aoff[q+1], moff[q+1] = uint32(len(a)), uint32(len(m))
		total += int(size[q])
	}
	a, m = append(a, 0), append(m, 0) // valid pointers for empty lists
	masks, nodes = append(masks, 0), append(nodes, 0xFFFFFFFF)
	par, dep := append(parent, 0), append(depth, 0)
	sz := append(size, 0)
	out, ooff := make([]uint32, total+1), make([]uint32, nreq+1)
	err := kxCheck(k.ctx, "kxpu_preferred_allocation_pcie", C.kxpu_preferred_allocation_pcie(k.ctx,
		(*C.uint64_t)(unsafe.Pointer(&masks[0])), (*C.uint32_t)(unsafe.Pointer(&nodes[0])), C.size_t(len(masks)-1),
		(*C.uint32_t)(unsafe.Pointer(&par[0])), (*C.uint8_t)(unsafe.Pointer(&dep[0])), C.size_t(len(parent)),
		(*C.uint32_t)(unsafe.Pointer(&aoff[0])), (*C.uint32_t)(unsafe.Pointer(&a[0])), (*C.uint32_t)(unsafe.Pointer(&moff[0])),
		(*C.uint32_t)(unsafe.Pointer(&m[0])), (*C.uint32_t)(unsafe.Pointer(&sz[0])), C.size_t(nreq),
		(*C.uint32_t)(unsafe.Pointer(&out[0])), (*C.uint32_t)(unsafe.Pointer(&ooff[0]))))
	res := make([][]uint32, nreq)
	for q := 0; err == nil && q < nreq; q++ {
		res[q] = out[ooff[q]:ooff[q+1]]
	}
	return res, err
}

// Runtime rediscovery (ABI v6).  After the walk and classify of a rediscovery, build one C.kxpu_snaprec per accepted
// function (key = PCI address, tag = the packed device id text) or mdev (key = UUID, tag = FNV-1a 64 of the type key),
// in walk order, and reconcile it against the previous snapshot: survivors keep their CDI index, everything else gets
// a fresh one from nextIndex on.  The returned snapshot (cur with the new indices) and next index are the input of the
// next rediscovery.  prev may be empty (nextIndex = 0 numbers by walk order, the start-up busIndex).
func (k *kxpu) reconcile(prev []C.kxpu_snaprec, nextIndex uint64, cur []C.kxpu_snaprec) (snap []C.kxpu_snaprec,
	curState, prevState []uint8, counts C.kxpu_reconcile_counts, err error) {
	idx := make([]uint64, len(cur)+1)
	curState, prevState = make([]uint8, len(cur)+1), make([]uint8, len(prev)+1)
	var pp, cp unsafe.Pointer
	if len(prev) > 0 {
		pp = unsafe.Pointer(&prev[0])
	}
	if len(cur) > 0 {
		cp = unsafe.Pointer(&cur[0])
	}
	err = kxCheck(k.ctx, "kxpu_reconcile", C.kxpu_reconcile(k.ctx, (*C.kxpu_snaprec)(pp), C.size_t(len(prev)),
		C.uint64_t(nextIndex), (*C.kxpu_snaprec)(cp), C.size_t(len(cur)), (*C.uint64_t)(unsafe.Pointer(&idx[0])),
		(*C.uint8_t)(unsafe.Pointer(&curState[0])), (*C.uint8_t)(unsafe.Pointer(&prevState[0])), &counts))
	if err != nil {
		return nil, nil, nil, counts, err
	}
	snap = append([]C.kxpu_snaprec(nil), cur...)
	for i := range snap {
		snap[i].index = C.uint64_t(idx[i])
	}
	return snap, curState[:len(cur)], prevState[:len(prev)], counts, nil
}

// Restart resume (ABI v13).  cdiParse / cdiParseMdev read back a CDI spec this library wrote: the records, in document
// order, of which kxpu_cdi_emit_kind / kxpu_cdi_emit_mdev write exactly these bytes; any other document is an error
// (KXPU_E_INVALID).  One call: len(doc) / KXPU_CDI_FRAG_MIN records hold every document.
func (k *kxpu) cdiParse(format int, doc []byte, kind string) ([]C.kxpu_cdidev, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	out := make([]C.kxpu_cdidev, len(doc)/C.KXPU_CDI_FRAG_MIN+1)
	var n C.size_t
	var dp *C.uint8_t
	if len(doc) > 0 {
		dp = (*C.uint8_t)(unsafe.Pointer(&doc[0]))
	}
	err := kxCheck(k.ctx, "kxpu_cdi_parse", C.kxpu_cdi_parse(k.ctx, C.int32_t(format), ck, dp, C.size_t(len(doc)), &out[0],
		C.size_t(len(out)), &n))
	if err != nil {
		return nil, err
	}
	return out[:n], nil
}

func (k *kxpu) cdiParseMdev(format int, doc []byte, kind string) ([]C.kxpu_mdevcdi, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	out := make([]C.kxpu_mdevcdi, len(doc)/C.KXPU_CDI_FRAG_MIN+1)
	var n C.size_t
	var dp *C.uint8_t
	if len(doc) > 0 {
		dp = (*C.uint8_t)(unsafe.Pointer(&doc[0]))
	}
	err := kxCheck(k.ctx, "kxpu_cdi_parse_mdev", C.kxpu_cdi_parse_mdev(k.ctx, C.int32_t(format), ck, dp, C.size_t(len(doc)),
		&out[0], C.size_t(len(out)), &n))
	if err != nil {
		return nil, err
	}
	return out[:n], nil
}

// VFIO cdevs (ABI v14).  cdiEmitCdev writes cdiEmitKind's document with each device's node /dev/vfio/devices/vfio<N>,
// N = devs[i].vfio_cdev (read from <bdf>/vfio-dev/vfio<N>); cdiParseCdev is its inverse and returns N in vfio_cdev.  A
// group-layout document is an error for cdiParseCdev, and a cdev document for cdiParse.
func (k *kxpu) cdiEmitCdev(format int, kind string, devs []C.kxpu_cdidev) ([]byte, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	var p *C.kxpu_cdidev
	if len(devs) > 0 {
		p = &devs[0]
	}
	var n C.size_t
	C.kxpu_cdi_emit_cdev(k.ctx, C.int32_t(format), ck, p, C.size_t(len(devs)), nil, 0, &n) // sizing call
	buf := make([]byte, n+1)
	err := kxCheck(k.ctx, "kxpu_cdi_emit_cdev", C.kxpu_cdi_emit_cdev(k.ctx, C.int32_t(format), ck, p, C.size_t(len(devs)),
		(*C.uint8_t)(unsafe.Pointer(&buf[0])), n, &n))
	return buf[:n], err
}

func (k *kxpu) cdiParseCdev(format int, doc []byte, kind string) ([]C.kxpu_cdidev, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	out := make([]C.kxpu_cdidev, len(doc)/C.KXPU_CDI_FRAG_MIN+1)
	var n C.size_t
	var dp *C.uint8_t
	if len(doc) > 0 {
		dp = (*C.uint8_t)(unsafe.Pointer(&doc[0]))
	}
	err := kxCheck(k.ctx, "kxpu_cdi_parse_cdev", C.kxpu_cdi_parse_cdev(k.ctx, C.int32_t(format), ck, dp, C.size_t(len(doc)),
		&out[0], C.size_t(len(out)), &n))
	if err != nil {
		return nil, err
	}
	return out[:n], nil
}

// VFIO cdevs of vGPUs (additions to ABI v14, detected by symbol).  cdiEmitMdevCdev writes cdiEmitMdev's document for
// devs[i].dev with each device's node /dev/vfio/devices/vfio<N>, N = devs[i].vfio_cdev (read from
// <mdevBasePath>/<uuid>/vfio-dev/vfio<N>); cdiParseMdevCdev is its inverse and returns N in vfio_cdev.  Each of the four
// parsers refuses the other layouts' documents, except the zero-device document, which all of them accept.
func (k *kxpu) cdiEmitMdevCdev(format int, kind string, devs []C.kxpu_mdevcdev) ([]byte, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	var p *C.kxpu_mdevcdev
	if len(devs) > 0 {
		p = &devs[0]
	}
	var n C.size_t
	C.kxpu_cdi_emit_mdev_cdev(k.ctx, C.int32_t(format), ck, p, C.size_t(len(devs)), nil, 0, &n) // sizing call
	buf := make([]byte, n+1)
	err := kxCheck(k.ctx, "kxpu_cdi_emit_mdev_cdev", C.kxpu_cdi_emit_mdev_cdev(k.ctx, C.int32_t(format), ck, p,
		C.size_t(len(devs)), (*C.uint8_t)(unsafe.Pointer(&buf[0])), n, &n))
	return buf[:n], err
}

func (k *kxpu) cdiParseMdevCdev(format int, doc []byte, kind string) ([]C.kxpu_mdevcdev, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	out := make([]C.kxpu_mdevcdev, len(doc)/C.KXPU_CDI_FRAG_MIN+1)
	var n C.size_t
	var dp *C.uint8_t
	if len(doc) > 0 {
		dp = (*C.uint8_t)(unsafe.Pointer(&doc[0]))
	}
	err := kxCheck(k.ctx, "kxpu_cdi_parse_mdev_cdev", C.kxpu_cdi_parse_mdev_cdev(k.ctx, C.int32_t(format), ck, dp,
		C.size_t(len(doc)), &out[0], C.size_t(len(out)), &n))
	if err != nil {
		return nil, err
	}
	return out[:n], nil
}

// The spec of a class that serves vGPUs on SR-IOV VFs, with each VF's vGPU type (additions to ABI v14, detected by
// symbol).  cdiEmitVfVgpu writes cdiEmitKind's document (cdev: cdiEmitCdev's) for devs[i].dev with two more annotations
// per device, vgpu-type: "<type_id>" and vgpu-type-key: "<key>"; cdiParseVfVgpu is its inverse.  Written when indices
// are resumed across restarts, so that a restarted plugin reads back the names of the types it serves (a full GPU
// lists none in creatable_vgpu_types) and gives a VF whose type changed while it was down a fresh index.  The six CDI
// parsers refuse each other's documents, except the zero-device document, which all of them accept.
func (k *kxpu) cdiEmitVfVgpu(format int, kind string, devs []C.kxpu_vfvgpucdi) ([]byte, error) {
	return k.cdiEmitVfVgpuCall(format, kind, devs, false)
}

func (k *kxpu) cdiEmitVfVgpuCdev(format int, kind string, devs []C.kxpu_vfvgpucdi) ([]byte, error) {
	return k.cdiEmitVfVgpuCall(format, kind, devs, true)
}

func (k *kxpu) cdiEmitVfVgpuCall(format int, kind string, devs []C.kxpu_vfvgpucdi, cdev bool) ([]byte, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	var p *C.kxpu_vfvgpucdi
	if len(devs) > 0 {
		p = &devs[0]
	}
	// cgo calls a C function only by name, so each layout has its own call
	call := func(out *C.uint8_t, cap C.size_t, n *C.size_t) C.int32_t {
		if cdev {
			return C.kxpu_cdi_emit_vf_vgpu_cdev(k.ctx, C.int32_t(format), ck, p, C.size_t(len(devs)), out, cap, n)
		}
		return C.kxpu_cdi_emit_vf_vgpu(k.ctx, C.int32_t(format), ck, p, C.size_t(len(devs)), out, cap, n)
	}
	what := "kxpu_cdi_emit_vf_vgpu"
	if cdev {
		what = "kxpu_cdi_emit_vf_vgpu_cdev"
	}
	var n C.size_t
	call(nil, 0, &n) // sizing call
	buf := make([]byte, n+1)
	err := kxCheck(k.ctx, what, call((*C.uint8_t)(unsafe.Pointer(&buf[0])), n, &n))
	return buf[:n], err
}

func (k *kxpu) cdiParseVfVgpu(format int, doc []byte, kind string) ([]C.kxpu_vfvgpucdi, error) {
	return k.cdiParseVfVgpuCall(format, doc, kind, false)
}

func (k *kxpu) cdiParseVfVgpuCdev(format int, doc []byte, kind string) ([]C.kxpu_vfvgpucdi, error) {
	return k.cdiParseVfVgpuCall(format, doc, kind, true)
}

func (k *kxpu) cdiParseVfVgpuCall(format int, doc []byte, kind string, cdev bool) ([]C.kxpu_vfvgpucdi, error) {
	ck := C.CString(kind)
	defer C.free(unsafe.Pointer(ck))
	out := make([]C.kxpu_vfvgpucdi, len(doc)/C.KXPU_CDI_FRAG_MIN+1)
	var n C.size_t
	var dp *C.uint8_t
	if len(doc) > 0 {
		dp = (*C.uint8_t)(unsafe.Pointer(&doc[0]))
	}
	var rc C.int32_t
	what := "kxpu_cdi_parse_vf_vgpu"
	if cdev {
		what = "kxpu_cdi_parse_vf_vgpu_cdev"
		rc = C.kxpu_cdi_parse_vf_vgpu_cdev(k.ctx, C.int32_t(format), ck, dp, C.size_t(len(doc)), &out[0], C.size_t(len(out)), &n)
	} else {
		rc = C.kxpu_cdi_parse_vf_vgpu(k.ctx, C.int32_t(format), ck, dp, C.size_t(len(doc)), &out[0], C.size_t(len(out)), &n)
	}
	err := kxCheck(k.ctx, what, rc)
	if err != nil {
		return nil, err
	}
	return out[:n], nil
}

// cdiParseVgpuSpec: the records of a vGPU class's previous spec for the restart resume (resumeWalk's prev entries).  It
// is parsed with the layout the class uses now (mdevCdev: the cdev layout), then with the other one, so a class that
// switched mdevCdev across the restart keeps its indices; only the kxpu_mdevcdi part (uuid, group, index) is returned.
func (k *kxpu) cdiParseVgpuSpec(doc []byte, kind string, mdevCdev bool) ([]C.kxpu_mdevcdi, error) {
	viaCdev := func() ([]C.kxpu_mdevcdi, error) {
		recs, err := k.cdiParseMdevCdev(C.KXPU_FMT_YAML, doc, kind)
		if err != nil {
			return nil, err
		}
		out := make([]C.kxpu_mdevcdi, len(recs))
		for i := range recs {
			out[i] = recs[i].dev
		}
		return out, nil
	}
	viaGroup := func() ([]C.kxpu_mdevcdi, error) { return k.cdiParseMdev(C.KXPU_FMT_YAML, doc, kind) }
	first, second := viaGroup, viaCdev
	if mdevCdev {
		first, second = viaCdev, viaGroup
	}
	recs, err := first()
	if err != nil && strings.Contains(err.Error(), "invalid") {
		recs, err = second()
	}
	return recs, err
}

// The index state file of the restart resume: <cdiConfigPath>.kata-xpu-cdi-index, "pci <next>\nmdev <next>\n".  The CDI
// cache loads only *.json / *.yaml.  Write it (tmp + fsync + rename, only when its bytes change) whenever a next index
// grows, before any spec that names the new indices.
const indexStateName = ".kata-xpu-cdi-index"

func readIndexState(cdiConfigPath string) (pciNext, mdevNext uint64, ok bool) {
	b, err := os.ReadFile(cdiConfigPath + indexStateName)
	if err != nil {
		return 0, 0, false
	}
	var p, m uint64
	if n, err := fmt.Sscanf(string(b), "pci %d\nmdev %d\n", &p, &m); err != nil || n != 2 ||
		fmt.Sprintf("pci %d\nmdev %d\n", p, m) != string(b) {
		fmt.Fprintf(os.Stderr, "CDI index state %s: malformed, resuming without it\n", cdiConfigPath+indexStateName)
		return 0, 0, false
	}
	return p, m, true
}

// resumeWalk: the start-up reconcile of one walk against the previous specs.  prev holds one entry per parsed record
// (key = bdf or UUID, the parsed group, klass = the position of the class whose file it came from, tag 0, the parsed
// index), cur the first walk's entries in walk order (klass = the class of the entry's group, tag 0), stateNext the
// state file's value (0 without one).  fallback != "" (a file that did not parse, an index or key named twice, an index
// of 2^64-1) or a refused reconcile numbers the walk afresh from stateNext.  The caller rebuilds its maps with the
// returned indices and keeps the usual snapshot (real tags) and counts.next_index_out, exactly as Plugin::resumeIndices
// does in host/device_plugin.cpp.
func (k *kxpu) resumeWalk(prev []C.kxpu_snaprec, stateNext uint64, cur []C.kxpu_snaprec, fallback string) (
	index []uint64, counts C.kxpu_reconcile_counts, why string, err error) {
	next := stateNext
	for _, p := range prev {
		if uint64(p.index)+1 > next {
			next = uint64(p.index) + 1
		}
	}
	why = fallback
	for attempt := 0; attempt < 2; attempt++ {
		if why != "" {
			fmt.Fprintf(os.Stderr, "CDI index resume: %s; numbering this walk afresh from %d\n", why, stateNext)
			prev, next = nil, stateNext
		}
		var snap []C.kxpu_snaprec
		snap, _, _, counts, err = k.reconcile(prev, next, cur)
		if err == nil {
			index = make([]uint64, len(snap))
			for i := range snap {
				index[i] = uint64(snap[i].index)
			}
			return index, counts, why, nil
		}
		if why != "" || !strings.Contains(err.Error(), "invalid") {
			return nil, counts, why, err
		}
		why = "kxpu_reconcile refused the previous entries: " + err.Error()
	}
	return nil, counts, why, err
}

// DRA ResourceSlices (ABI v9).  One pool per class with a DRA driver, named after the node (NODE_NAME): devs holds one
// kxpu_dradev per published IOMMU group in walk order (groups with a viability blocker left out).  Returns the slices
// as JSON Lines, one object per line; the caller POSTs each line to /apis/resource.k8s.io/v1/resourceslices and then
// deletes the slices of its driver and node with an older spec.pool.generation.
//
// DRA device taints (ABI v11, v12): since == nil publishes no taints.  Otherwise since holds one or three times per
// device, device-major, -1 where the device does not carry that taint, for the first one or all three entries of the
// table [<driver>/unhealthy=vfio-device-missing, <driver>/pcie-aer=fatal, <driver>/pcie-aer=nonfatal], all
// NoSchedule: a missing device node keeps new claims away but must not evict a VM that holds the group open.  A device
// carries at most one of the two pcie-aer values.  With taints a slice holds 64 devices.
func (k *kxpu) draSlices(driver, node string, generation uint64, devs []C.kxpu_dradev, since []int64) ([]string, error) {
	var p *C.kxpu_dradev
	if len(devs) > 0 {
		p = &devs[0]
	}
	return k.slices("kxpu_dra_slices_taints", driver, node, len(devs), since, func(cd, cn *C.char, tab *C.kxpu_dra_taint,
		nt C.size_t, cs *C.int64_t, out *C.uint8_t, capacity C.size_t, n *C.size_t, off *C.uint64_t, ns *C.size_t) C.int32_t {
		return C.kxpu_dra_slices_taints(k.ctx, cd, cn, cn, C.uint64_t(generation), p, C.size_t(len(devs)), tab, nt, cs, out,
			capacity, n, off, ns)
	})
}

// DRA ResourceSlices of vGPUs (ABI v10).  One pool per vGPU class with a DRA driver, named after the node: devs holds one
// kxpu_dramdev per mdevMap group of the class in walk order.  Tainted, published and replaced exactly as draSlices'
// output.
func (k *kxpu) draSlicesMdev(driver, node string, generation uint64, devs []C.kxpu_dramdev, since []int64) ([]string, error) {
	var p *C.kxpu_dramdev
	if len(devs) > 0 {
		p = &devs[0]
	}
	return k.slices("kxpu_dra_slices_mdev_taints", driver, node, len(devs), since, func(cd, cn *C.char,
		tab *C.kxpu_dra_taint, nt C.size_t, cs *C.int64_t, out *C.uint8_t, capacity C.size_t, n *C.size_t, off *C.uint64_t,
		ns *C.size_t) C.int32_t {
		return C.kxpu_dra_slices_mdev_taints(k.ctx, cd, cn, cn, C.uint64_t(generation), p, C.size_t(len(devs)), tab, nt, cs,
			out, capacity, n, off, ns)
	})
}

// DRA ResourceSlices of vGPUs on SR-IOV VFs (an addition to ABI v14).  One pool per vfVgpu class with a vgpuDraDriver,
// named after the node: devs holds one kxpu_dravfvgpu per published VF group of the class in walk order, and generation
// is the PCI walk's pool generation.  Tainted, published and replaced exactly as draSlices' output.
func (k *kxpu) draSlicesVfVgpu(driver, node string, generation uint64, devs []C.kxpu_dravfvgpu, since []int64) ([]string, error) {
	var p *C.kxpu_dravfvgpu
	if len(devs) > 0 {
		p = &devs[0]
	}
	return k.slices("kxpu_dra_slices_vf_vgpu", driver, node, len(devs), since, func(cd, cn *C.char,
		tab *C.kxpu_dra_taint, nt C.size_t, cs *C.int64_t, out *C.uint8_t, capacity C.size_t, n *C.size_t, off *C.uint64_t,
		ns *C.size_t) C.int32_t {
		return C.kxpu_dra_slices_vf_vgpu(k.ctx, cd, cn, cn, C.uint64_t(generation), p, C.size_t(len(devs)), tab, nt, cs,
			out, capacity, n, off, ns)
	})
}

// DRA ResourceSlices of mdev vGPUs whose parents may be SR-IOV VFs (an addition to ABI v14, detected by symbol).  With
// vgpuSriovAware a vGPU class's pool is published through this call instead of draSlicesMdev: devs holds one
// kxpu_dramdevpf per mdevMap group of the class in walk order, its PF's address and device id next to the mdev record
// (both empty for an mdev on a PF, which then gives draSlicesMdev's bytes).  Tainted, published and replaced exactly as
// draSlicesMdev's output.
func (k *kxpu) draSlicesMdevPf(driver, node string, generation uint64, devs []C.kxpu_dramdevpf, since []int64) ([]string, error) {
	var p *C.kxpu_dramdevpf
	if len(devs) > 0 {
		p = &devs[0]
	}
	return k.slices("kxpu_dra_slices_mdev_pf", driver, node, len(devs), since, func(cd, cn *C.char,
		tab *C.kxpu_dra_taint, nt C.size_t, cs *C.int64_t, out *C.uint8_t, capacity C.size_t, n *C.size_t, off *C.uint64_t,
		ns *C.size_t) C.int32_t {
		return C.kxpu_dra_slices_mdev_pf(k.ctx, cd, cn, cn, C.uint64_t(generation), p, C.size_t(len(devs)), tab, nt, cs,
			out, capacity, n, off, ns)
	})
}

// DRA ResourceSlices of passthrough devices that may be SR-IOV VFs (an addition to ABI v14, detected by symbol).  With
// sriovPfAware a passthrough class's pool is published through this call instead of draSlices: devs holds one
// kxpu_dradevpf per published group of the class in walk order, the PF's address (pfOf of the group's first member,
// from sriov) and the PF's device id next to the record (both empty for a function that is no VF, which then gives
// draSlices' bytes).  Tainted, published and replaced exactly as draSlices' output.
func (k *kxpu) draSlicesPf(driver, node string, generation uint64, devs []C.kxpu_dradevpf, since []int64) ([]string, error) {
	var p *C.kxpu_dradevpf
	if len(devs) > 0 {
		p = &devs[0]
	}
	return k.slices("kxpu_dra_slices_pf", driver, node, len(devs), since, func(cd, cn *C.char,
		tab *C.kxpu_dra_taint, nt C.size_t, cs *C.int64_t, out *C.uint8_t, capacity C.size_t, n *C.size_t, off *C.uint64_t,
		ns *C.size_t) C.int32_t {
		return C.kxpu_dra_slices_pf(k.ctx, cd, cn, cn, C.uint64_t(generation), p, C.size_t(len(devs)), tab, nt, cs,
			out, capacity, n, off, ns)
	})
}

// draPcieConfig is Plugin::draPcieDomain: empty (default) publishes every passthrough pool as before; a lowercase DNS
// subdomain of at most 63 bytes, not kubernetes.io or k8s.io nor under either, and only with a draDriver on some
// passthrough class, publishes every passthrough pool through draSlicesPcie.
type draPcieConfig struct {
	DraPcieDomain string
}

// DRA ResourceSlices with each device's PCIe root port and switch (an addition to ABI v14, detected by symbol).  devs
// holds one kxpu_dradevpcie per published group in walk order: the kxpu_dradevpf of draSlicesPf (its physfn fields
// filled only with sriovPfAware) and the group's two keys from pciePorts.  Tainted, published and replaced exactly as
// draSlices' output; with every key C.KXPU_PCIE_NO_KEY the bytes are draSlicesPf's.
func (k *kxpu) draSlicesPcie(driver, node string, generation uint64, domain string, devs []C.kxpu_dradevpcie,
	since []int64) ([]string, error) {
	var p *C.kxpu_dradevpcie
	if len(devs) > 0 {
		p = &devs[0]
	}
	cdom := C.CString(domain)
	defer C.free(unsafe.Pointer(cdom))
	return k.slices("kxpu_dra_slices_pcie", driver, node, len(devs), since, func(cd, cn *C.char,
		tab *C.kxpu_dra_taint, nt C.size_t, cs *C.int64_t, out *C.uint8_t, capacity C.size_t, n *C.size_t, off *C.uint64_t,
		ns *C.size_t) C.int32_t {
		return C.kxpu_dra_slices_pcie(k.ctx, cd, cn, cn, C.uint64_t(generation), cdom, p, C.size_t(len(devs)), tab, nt, cs,
			out, capacity, n, off, ns)
	})
}

// draVgpuPcieConfig is Plugin::draVgpuPcie: false (default) publishes the vGPU pools as before; true, only with
// DraPcieDomain set and a vGPU class that publishes DRA, publishes them through draSlicesMdevPcie and
// draSlicesVfVgpuPcie under DraPcieDomain's names.
type draVgpuPcieConfig struct {
	DraVgpuPcie bool
}

// DRA ResourceSlices of mdev vGPUs with their parent GPU's PCIe root port and switch (an addition to ABI v14, detected
// by symbol).  devs: one kxpu_dramdevpcie per published group, draSlicesMdevPf's record and pciePortsMdev's keys; with
// every key C.KXPU_PCIE_NO_KEY the bytes are draSlicesMdevPf's.
func (k *kxpu) draSlicesMdevPcie(driver, node string, generation uint64, domain string, devs []C.kxpu_dramdevpcie,
	since []int64) ([]string, error) {
	var p *C.kxpu_dramdevpcie
	if len(devs) > 0 {
		p = &devs[0]
	}
	cdom := C.CString(domain)
	defer C.free(unsafe.Pointer(cdom))
	return k.slices("kxpu_dra_slices_mdev_pcie", driver, node, len(devs), since, func(cd, cn *C.char,
		tab *C.kxpu_dra_taint, nt C.size_t, cs *C.int64_t, out *C.uint8_t, capacity C.size_t, n *C.size_t, off *C.uint64_t,
		ns *C.size_t) C.int32_t {
		return C.kxpu_dra_slices_mdev_pcie(k.ctx, cd, cn, cn, C.uint64_t(generation), cdom, p, C.size_t(len(devs)), tab, nt,
			cs, out, capacity, n, off, ns)
	})
}

// DRA ResourceSlices of vGPUs on VFs with their PCIe ports (an addition to ABI v14, detected by symbol).  devs: one
// kxpu_dravfvgpupcie per published group, draSlicesVfVgpu's record and the keys pciePorts gave the VF's group; with every
// key C.KXPU_PCIE_NO_KEY the bytes are draSlicesVfVgpu's.
func (k *kxpu) draSlicesVfVgpuPcie(driver, node string, generation uint64, domain string, devs []C.kxpu_dravfvgpupcie,
	since []int64) ([]string, error) {
	var p *C.kxpu_dravfvgpupcie
	if len(devs) > 0 {
		p = &devs[0]
	}
	cdom := C.CString(domain)
	defer C.free(unsafe.Pointer(cdom))
	return k.slices("kxpu_dra_slices_vf_vgpu_pcie", driver, node, len(devs), since, func(cd, cn *C.char,
		tab *C.kxpu_dra_taint, nt C.size_t, cs *C.int64_t, out *C.uint8_t, capacity C.size_t, n *C.size_t, off *C.uint64_t,
		ns *C.size_t) C.int32_t {
		return C.kxpu_dra_slices_vf_vgpu_pcie(k.ctx, cd, cn, cn, C.uint64_t(generation), cdom, p, C.size_t(len(devs)), tab,
			nt, cs, out, capacity, n, off, ns)
	})
}

// the two-call sizing of one slice call, the table and the times in C memory; the table width is len(since) / nDevs
func (k *kxpu) slices(what, driver, node string, nDevs int, since []int64, call func(cd, cn *C.char,
	tab *C.kxpu_dra_taint, nt C.size_t, cs *C.int64_t, out *C.uint8_t, capacity C.size_t, n *C.size_t, off *C.uint64_t,
	ns *C.size_t) C.int32_t) ([]string, error) {
	nt := 1
	if since != nil && nDevs > 0 {
		nt = len(since) / nDevs
	}
	if since != nil && (nt < 1 || nt > 3 || len(since) != nt*nDevs) {
		return nil, fmt.Errorf("%s: %d taint times for %d devices", what, len(since), nDevs)
	}
	strs := []*C.char{C.CString(driver), C.CString(node), C.CString(driver + "/unhealthy"), C.CString("vfio-device-missing"),
		C.CString(driver + "/pcie-aer"), C.CString("fatal"), C.CString("nonfatal"), C.CString("NoSchedule")}
	for _, s := range strs {
		defer C.free(unsafe.Pointer(s))
	}
	tab := (*C.kxpu_dra_taint)(C.malloc(C.size_t(3 * unsafe.Sizeof(C.kxpu_dra_taint{}))))
	defer C.free(unsafe.Pointer(tab))
	t := unsafe.Slice(tab, 3)
	t[0] = C.kxpu_dra_taint{key: strs[2], value: strs[3], effect: strs[7]}
	t[1] = C.kxpu_dra_taint{key: strs[4], value: strs[5], effect: strs[7]}
	t[2] = C.kxpu_dra_taint{key: strs[4], value: strs[6], effect: strs[7]}
	var cs *C.int64_t // nil: taint_since NULL, the untainted slices
	if since != nil {
		cs = (*C.int64_t)(C.malloc(C.size_t(8 * (len(since) + 1))))
		defer C.free(unsafe.Pointer(cs))
		copy(unsafe.Slice((*int64)(unsafe.Pointer(cs)), len(since)), since)
	}
	var n, ns C.size_t
	if rc := call(strs[0], strs[1], tab, C.size_t(nt), cs, nil, 0, &n, nil, &ns); rc != C.KXPU_E_NOSPACE { // sizing call
		return nil, kxCheck(k.ctx, what, rc)
	}
	buf := make([]byte, n)
	off := make([]uint64, ns+1)
	if err := kxCheck(k.ctx, what, call(strs[0], strs[1], tab, C.size_t(nt), cs, (*C.uint8_t)(unsafe.Pointer(&buf[0])), n, &n,
		(*C.uint64_t)(unsafe.Pointer(&off[0])), &ns)); err != nil {
		return nil, err
	}
	lines := make([]string, ns)
	for s := range lines {
		lines[s] = string(buf[off[s] : off[s+1]-1]) // without the '\n'
	}
	return lines, nil
}

// PCIe AER health (ABI v12).  text holds every file the host read (ReadFile of <bdf>/aer_dev_fatal and aer_dev_nonfatal,
// at most 4097 bytes each; an mdev reads its parent's, a failed read is an empty file); fileOff / fileLen are 2n entries,
// the fatal file of record i at 2i.  groupOff / groupMembers: the groups.  Returns each group's KXPU_AER_* bits.
func (k *kxpu) aerHealth(text []byte, fileOff []uint64, fileLen []uint32, fatalLimit, nonfatalLimit uint64,
	groupOff, groupMembers []uint32) ([]uint8, error) {
	if len(fileOff) != len(fileLen) || len(fileOff)%2 != 0 || len(groupOff) == 0 {
		return nil, fmt.Errorf("kxpu_aer_health: %d offsets, %d lengths, %d group offsets", len(fileOff), len(fileLen), len(groupOff))
	}
	nG := len(groupOff) - 1
	// the inputs go through C memory: cgo forbids passing several Go pointers that the callee keeps together
	ct := (*C.uint8_t)(C.malloc(C.size_t(len(text) + 1)))
	defer C.free(unsafe.Pointer(ct))
	copy(unsafe.Slice((*byte)(unsafe.Pointer(ct)), len(text)), text)
	co := (*C.uint64_t)(C.malloc(C.size_t(8 * (len(fileOff) + 1))))
	defer C.free(unsafe.Pointer(co))
	copy(unsafe.Slice((*uint64)(unsafe.Pointer(co)), len(fileOff)), fileOff)
	cl := (*C.uint32_t)(C.malloc(C.size_t(4 * (len(fileLen) + 1))))
	defer C.free(unsafe.Pointer(cl))
	copy(unsafe.Slice((*uint32)(unsafe.Pointer(cl)), len(fileLen)), fileLen)
	cg := (*C.uint32_t)(C.malloc(C.size_t(4 * (len(groupOff) + len(groupMembers)))))
	defer C.free(unsafe.Pointer(cg))
	g := unsafe.Slice((*uint32)(unsafe.Pointer(cg)), len(groupOff)+len(groupMembers))
	copy(g, groupOff)
	copy(g[len(groupOff):], groupMembers)
	out := (*C.uint8_t)(C.malloc(C.size_t(nG + 1)))
	defer C.free(unsafe.Pointer(out))
	if err := kxCheck(k.ctx, "kxpu_aer_health", C.kxpu_aer_health(k.ctx, ct, C.size_t(len(text)), co, cl,
		C.size_t(len(fileOff)/2), C.uint64_t(fatalLimit), C.uint64_t(nonfatalLimit), cg,
		(*C.uint32_t)(unsafe.Add(unsafe.Pointer(cg), 4*len(groupOff))), C.size_t(nG), nil, out)); err != nil {
		return nil, err
	}
	return append([]uint8(nil), unsafe.Slice((*uint8)(unsafe.Pointer(out)), nG)...), nil
}

// SR-IOV virtual functions (additions to ABI v14, detected by symbol).  With sriovAware on, the PCI walk also reads
// os.Readlink(<bdf>/physfn) (its basename) and the first 8 bytes of <bdf>/sriov_numvfs of every candidate of a
// passthrough class into a kxpu_sriovrec at the record's index (sriovRecord); a missing link or file is not an error.
// After classify, sriov gives each group's first blocking member: a group with one is sent Unhealthy, refused by
// Allocate and NodePrepareResources, and left out of the CDI spec and the DRA pool.  The reason names the function:
// "<vf> needs the VF token of <pf> (bound to <driver>)" when pfOf[i] is set and that PF's driver is a class driver, else
// "<pf> has <k> VFs enabled".  With pcieTopology on too, the forest comes from pcieTreeSriov(..., pfOf).

// the kxpu_sriovrec of one function from its two reads (physfnErr / numvfsErr: a failure other than "does not exist")
func sriovRecord(physfn string, physfnErr bool, numvfs []byte, numvfsErr bool) C.kxpu_sriovrec {
	var s C.kxpu_sriovrec
	if len(physfn) < len(s.physfn) {
		for i := 0; i < len(physfn); i++ {
			s.physfn[i] = C.char(physfn[i])
		}
	} else {
		physfnErr = true // no PCI address is this long
	}
	for i := 0; i < len(numvfs) && i < len(s.numvfs_txt); i++ {
		s.numvfs_txt[i] = C.uint8_t(numvfs[i])
	}
	n := len(numvfs)
	if n > len(s.numvfs_txt) {
		n = len(s.numvfs_txt) + 1
	}
	s.numvfs_len = C.uint8_t(n)
	if physfnErr {
		s.flags |= C.KXPU_SR_PHYSFN_ERR
	}
	if numvfsErr {
		s.flags |= C.KXPU_SR_NUMVFS_ERR
	}
	return s
}

// the SR-IOV verdict of a walk: recs / srs at the same indices, rules and the CSR (gids, goff, gmem) of its classify call.
// pfOf and numvfs have one entry per record, gsriov one per group (C.KXPU_VIABLE: served).
// mdevPf: each mdev's PF in the PCI walk (kxpu_mdev_pf, an addition to ABI v14).  recs: the PCI walk's records, which
// runs first; mrecs / msrs: the mdev walk's records and their physfn reads (readLink(<uuid>/../physfn), basename, in a
// kxpu_sriovrec whose numvfs fields stay zero).  pfOf[i] is a record index or KXPU_NO_PF.
func (k *kxpu) mdevPf(recs []C.kxpu_devrec, mrecs []C.kxpu_mdevrec, msrs []C.kxpu_sriovrec) ([]uint32, error) {
	n, m := len(recs), len(mrecs)
	pfOf := make([]uint32, m+1)
	var r *C.kxpu_devrec
	var mr *C.kxpu_mdevrec
	var ms *C.kxpu_sriovrec
	if n > 0 {
		r = &recs[0]
	}
	if m > 0 {
		mr, ms = &mrecs[0], &msrs[0]
	}
	err := kxCheck(k.ctx, "kxpu_mdev_pf", C.kxpu_mdev_pf(k.ctx, r, C.size_t(n), mr, ms, C.size_t(m),
		(*C.uint32_t)(unsafe.Pointer(&pfOf[0]))))
	return pfOf[:m], err
}

func (k *kxpu) sriov(rules []C.kxpu_xpu_rule, recs []C.kxpu_devrec, srs []C.kxpu_sriovrec, gids, goff, gmem []uint32) (pfOf,
	numvfs, gsriov []uint32, err error) {
	n, nGroups := len(recs), len(goff)-1
	pfOf, numvfs, gsriov = make([]uint32, n+1), make([]uint32, n+1), make([]uint32, nGroups+1)
	var r *C.kxpu_devrec
	var s *C.kxpu_sriovrec
	if n > 0 {
		r, s = &recs[0], &srs[0]
	}
	gi, gm := append(gids, 0), append(gmem, 0) // valid pointers for an empty walk
	err = kxCheck(k.ctx, "kxpu_sriov", C.kxpu_sriov(k.ctx, &rules[0], C.size_t(len(rules)), r, s, C.size_t(n),
		(*C.uint32_t)(unsafe.Pointer(&gi[0])), (*C.uint32_t)(unsafe.Pointer(&goff[0])), (*C.uint32_t)(unsafe.Pointer(&gm[0])),
		C.size_t(nGroups), (*C.uint32_t)(unsafe.Pointer(&pfOf[0])), (*C.uint32_t)(unsafe.Pointer(&numvfs[0])),
		(*C.uint32_t)(unsafe.Pointer(&gsriov[0]))))
	return pfOf[:n], numvfs[:n], gsriov[:nGroups], err
}

// Resets between tenants (an addition to ABI v14, detected by symbol).  With resetCheck on, the PCI walk also reads the
// entry link of every entry (pciPath), the driver link of every entry whose driver the class test did not read (and the
// iommu_group link of one bound to a class driver), and, for every candidate of a passthrough class, the first
// KXPU_RESET_FILE_MAX+1 bytes of <bdf>/reset_method, or when that does not exist whether <bdf>/reset exists
// (resetRecord).  After classify, resetCheck gives each group's reset blocker: a group with one is sent Unhealthy,
// refused by Allocate and NodePrepareResources, and left out of the CDI spec and every DRA pool, with the reason naming
// the function (methods[i] != 0: the methods resetMethods does not accept; else setVerdict[i]: a root bus, an unknown
// path, or the record on its bus that is bound to another driver, unbound, or in another group).

// the kxpu_resetrec of one candidate: text of reset_method (absent: no such file; readErr: any other failure), and
// legacy: <bdf>/reset exists (read only when reset_method is absent)
func resetRecord(text []byte, absent, readErr, legacy bool) C.kxpu_resetrec {
	var r C.kxpu_resetrec
	for i := 0; i < len(text) && i < len(r.txt); i++ {
		r.txt[i] = C.uint8_t(text[i])
	}
	n := len(text)
	if n > len(r.txt) {
		n = len(r.txt) + 1
	}
	r.len = C.uint8_t(n)
	if readErr {
		r.flags |= C.KXPU_RS_READ_ERR
	} else if absent {
		r.flags |= C.KXPU_RS_ABSENT
		if legacy {
			r.flags |= C.KXPU_RS_LEGACY
		}
	}
	return r
}

// the reset verdict of a walk: recs / paths / rrs at the same indices, the rules and CSR (goff, gmem) of its classify call,
// allow the KXPU_RM_* bits of resetMethods.  methods and setVerdict have one entry per record, greset one per group
// (C.KXPU_VIABLE: served).
func (k *kxpu) resetCheck(rules []C.kxpu_xpu_rule, recs []C.kxpu_devrec, paths []C.kxpu_pcipath, rrs []C.kxpu_resetrec,
	allow uint32, goff, gmem []uint32) (methods []uint8, setVerdict, greset []uint32, err error) {
	n, nGroups := len(recs), len(goff)-1
	methods, setVerdict, greset = make([]uint8, n+1), make([]uint32, n+1), make([]uint32, nGroups+1)
	var r *C.kxpu_devrec
	var pp *C.kxpu_pcipath
	var rr *C.kxpu_resetrec
	if n > 0 {
		r, pp, rr = &recs[0], &paths[0], &rrs[0]
	}
	gm := append(gmem, 0) // a valid pointer for an empty walk
	err = kxCheck(k.ctx, "kxpu_reset_check", C.kxpu_reset_check(k.ctx, &rules[0], C.size_t(len(rules)), r, pp, rr,
		C.size_t(n), C.uint32_t(allow), (*C.uint32_t)(unsafe.Pointer(&goff[0])), (*C.uint32_t)(unsafe.Pointer(&gm[0])),
		C.size_t(nGroups), (*C.uint8_t)(unsafe.Pointer(&methods[0])), (*C.uint32_t)(unsafe.Pointer(&setVerdict[0])),
		(*C.uint32_t)(unsafe.Pointer(&greset[0]))))
	return methods[:n], setVerdict[:n], greset[:nGroups], err
}

// Prometheus metrics (an addition to ABI v14, detected by symbol).  metricsDevices writes the device families of the
// text kxpu.h specifies (kata_xpu_device_healthy, _unhealthy_reason, kata_xpu_pcie_aer_errors) from one
// C.kxpu_metricdev per device and one C.kxpu_metricreason per reason, their strings in one byte table; metricsText
// appends the host's counters.  A host serves it on GET /metrics (INTEGRATION.md).
func (k *kxpu) metricsDevices(devs []C.kxpu_metricdev, strs []byte, reasons []C.kxpu_metricreason) ([]byte, error) {
	if len(devs) == 0 {
		return nil, nil
	}
	var s *C.uint8_t // NULL for an empty table: the caller's slices are only read
	var r *C.kxpu_metricreason
	if len(strs) > 0 {
		s = (*C.uint8_t)(unsafe.Pointer(&strs[0]))
	}
	if len(reasons) > 0 {
		r = &reasons[0]
	}
	call := func(out *C.uint8_t, cap C.size_t, n *C.size_t) C.int32_t {
		return C.kxpu_metrics_devices(k.ctx, &devs[0], C.size_t(len(devs)), s, C.size_t(len(strs)), r,
			C.size_t(len(reasons)), out, cap, n)
	}
	var n C.size_t
	if rc := call(nil, 0, &n); rc != C.KXPU_OK && rc != C.KXPU_E_NOSPACE { // sizing call
		return nil, kxCheck(k.ctx, "kxpu_metrics_devices", rc)
	}
	buf := make([]byte, n+1)
	err := kxCheck(k.ctx, "kxpu_metrics_devices", call((*C.uint8_t)(unsafe.Pointer(&buf[0])), n, &n))
	return buf[:n], err
}

// metricsCounters: the host's process counters, in the order and with the headers of kxpu.h
type metricsCounters struct {
	AerReads, CdevReads, SriovReads, ResetReads, VfVgpuReads uint64
	LiveValidations, SnapshotValidations                    uint64
}

func metricsText(device []byte, c metricsCounters) []byte {
	out := append([]byte(nil), device...)
	out = append(out, C.KXPU_METRICS_READS_HEAD...)
	for _, f := range []struct {
		name string
		v    uint64
	}{{"aer_dev", c.AerReads}, {"vfio-dev", c.CdevReads}, {"sriov", c.SriovReads}, {"reset", c.ResetReads},
		{"nvidia", c.VfVgpuReads}} {
		out = append(out, fmt.Sprintf("kata_xpu_sysfs_reads_total{file=%q} %d\n", f.name, f.v)...)
	}
	out = append(out, C.KXPU_METRICS_VALIDATIONS_HEAD...)
	out = append(out, fmt.Sprintf("kata_xpu_allocate_validations_total{path=\"live\"} %d\n", c.LiveValidations)...)
	out = append(out, fmt.Sprintf("kata_xpu_allocate_validations_total{path=\"snapshot\"} %d\n", c.SnapshotValidations)...)
	return out
}

// pcieTree with every VF below its PF (pfOf: sriov's)
func (k *kxpu) pcieTreeSriov(recs []C.kxpu_devrec, paths []C.kxpu_pcipath, goff, gmem []uint32, nGroups int,
	pfOf []uint32) (gnode, parent []uint32, depth []uint8, err error) {
	capN := 8*nGroups + 1
	gnode, parent, depth = make([]uint32, nGroups+1), make([]uint32, capN), make([]uint8, capN)
	key := make([]uint64, capN)
	var nn C.uint32_t
	var r unsafe.Pointer
	var pp *C.kxpu_pcipath
	pf := append(pfOf, 0) // a valid pointer for an empty walk
	if len(recs) > 0 {
		r, pp = unsafe.Pointer(&recs[0]), &paths[0]
	}
	gm := append(gmem, 0)
	err = kxCheck(k.ctx, "kxpu_pcie_tree_sriov", C.kxpu_pcie_tree_sriov(k.ctx, (*C.kxpu_devrec)(r), pp, C.size_t(len(recs)),
		(*C.uint32_t)(unsafe.Pointer(&goff[0])), (*C.uint32_t)(unsafe.Pointer(&gm[0])), C.size_t(nGroups),
		(*C.uint32_t)(unsafe.Pointer(&gnode[0])), (*C.uint64_t)(unsafe.Pointer(&key[0])),
		(*C.uint32_t)(unsafe.Pointer(&parent[0])), (*C.uint8_t)(unsafe.Pointer(&depth[0])), &nn,
		(*C.uint32_t)(unsafe.Pointer(&pf[0]))))
	return gnode[:nGroups], parent[:nn], depth[:nn], err
}

// PCIe forest of the mdev walk (addition to ABI v14, detected by symbol).  With vgpuPcieTopology on, the mdev walk runs
// os.Readlink(<mdevBasePath>/<uuid>) per entry that got as far as its iommu_group link (the read the vGPU DRA pool
// already does) and keeps pciPath of the target; after classifyMdev, pcieTreeMdev builds the forest on the classify
// CSR, every vGPU pluginapi.Device keeps its group's node, and GetPreferredAllocation of a vGPU plugin calls
// preferredAllocationPcie with this forest (passthrough plugins keep the PCI walk's).  An mdev's parent function is the
// deepest node of its chain, so a request is packed under one GPU, then one switch.
func (k *kxpu) pcieTreeMdev(recs []C.kxpu_mdevrec, paths []C.kxpu_pcipath, goff, gmem []uint32, nGroups int) (gnode,
	parent []uint32, depth []uint8, err error) {
	capN := 8*nGroups + 1
	gnode, parent, depth = make([]uint32, nGroups+1), make([]uint32, capN), make([]uint8, capN)
	key := make([]uint64, capN)
	var nn C.uint32_t
	var r unsafe.Pointer
	var pp *C.kxpu_pcipath
	if len(recs) > 0 {
		r, pp = unsafe.Pointer(&recs[0]), &paths[0]
	}
	gm := append(gmem, 0) // a valid pointer for an empty walk
	err = kxCheck(k.ctx, "kxpu_pcie_tree_mdev", C.kxpu_pcie_tree_mdev(k.ctx, (*C.kxpu_mdevrec)(r), pp, C.size_t(len(recs)),
		(*C.uint32_t)(unsafe.Pointer(&goff[0])), (*C.uint32_t)(unsafe.Pointer(&gm[0])), C.size_t(nGroups),
		(*C.uint32_t)(unsafe.Pointer(&gnode[0])), (*C.uint64_t)(unsafe.Pointer(&key[0])),
		(*C.uint32_t)(unsafe.Pointer(&parent[0])), (*C.uint8_t)(unsafe.Pointer(&depth[0])), &nn))
	return gnode[:nGroups], parent[:nn], depth[:nn], err
}

// vGPUs on SR-IOV virtual functions (additions to ABI v14, detected by symbol).  On a host with NVIDIA's
// vendor-specific VFIO framework each vGPU is a VF whose profile is <vf>/nvidia/current_vgpu_type; include/kxpu.h lists
// the facts this rests on as [assumed].  After the PCI walk, read current_vgpu_type (the first 16 bytes) and
// creatable_vgpu_types of every VF (a record with a physfn link) whose vendor and driver match a class that serves
// vGPUs on VFs; vfVgpuTypes joins each VF's type ID to a name and returns its key row, and classifyVfVgpu then gives
// one device-map entry per (class, type key).  This code was not compiled: the image has no Go toolchain.

// the kxpu_vfvgpurec of one VF from its current_vgpu_type read (curErr: the read failed, "does not exist" included)
func vfVgpuRecord(cur []byte, curErr bool) C.kxpu_vfvgpurec {
	var r C.kxpu_vfvgpurec
	r.flags = C.KXPU_VT_READ
	if curErr {
		r.flags |= C.KXPU_VT_CUR_ERR
		return r
	}
	for i := 0; i < len(cur) && i < len(r.cur_txt); i++ {
		r.cur_txt[i] = C.uint8_t(cur[i])
	}
	l := len(cur)
	if l > 16 {
		l = 17
	}
	r.cur_len = C.uint8_t(l)
	return r
}

// the type join: recs one side record per walk record, tables the name tables in priority order (the class's
// configured names, then every read creatable_vgpu_types in walk order, then the names learned in earlier walks).
// Returns one key row, type ID and status (C.KXPU_VT_*) per record.
func (k *kxpu) vfVgpuTypes(recs []C.kxpu_vfvgpurec, tables [][]byte) (keys []C.kxpu_vgpukey, typeID []uint32,
	status []uint8, err error) {
	n := len(recs)
	keys, typeID, status = make([]C.kxpu_vgpukey, n+1), make([]uint32, n+1), make([]uint8, n+1)
	off := make([]uint64, len(tables)+1)
	var blob []byte
	for i, t := range tables {
		blob = append(blob, t...)
		off[i+1] = uint64(len(blob))
	}
	blob = append(blob, 0) // a valid pointer for an empty blob
	var r *C.kxpu_vfvgpurec
	if n > 0 {
		r = &recs[0]
	}
	err = kxCheck(k.ctx, "kxpu_vf_vgpu_types", C.kxpu_vf_vgpu_types(k.ctx, r, C.size_t(n),
		(*C.uint8_t)(unsafe.Pointer(&blob[0])), (*C.uint64_t)(unsafe.Pointer(&off[0])), C.size_t(len(tables)), &keys[0],
		(*C.uint32_t)(unsafe.Pointer(&typeID[0])), (*C.uint8_t)(unsafe.Pointer(&status[0]))))
	return keys[:n], typeID[:n], status[:n], err
}

// the drift check: recs the re-read side records of the served VFs, was their walk's type IDs, one one-member group per
// VF.  Returns per record the type read back and its status (C.KXPU_VD_*), and per group the position of its first
// drifted member or C.KXPU_VD_STEADY.
func (k *kxpu) vfVgpuDrift(recs []C.kxpu_vfvgpurec, was []uint32, groupOff, groupMembers []uint32) (typeNow []uint32,
	status []uint8, first []uint32, err error) {
	n, g := len(recs), len(groupOff)-1
	typeNow, status, first = make([]uint32, n+1), make([]uint8, n+1), make([]uint32, g+1)
	was = append(was, 0)                   // valid pointers for n == 0
	groupMembers = append(groupMembers, 0) // and for no members
	var r *C.kxpu_vfvgpurec
	if n > 0 {
		r = &recs[0]
	}
	err = kxCheck(k.ctx, "kxpu_vf_vgpu_drift", C.kxpu_vf_vgpu_drift(k.ctx, r, (*C.uint32_t)(unsafe.Pointer(&was[0])),
		C.size_t(n), (*C.uint32_t)(unsafe.Pointer(&groupOff[0])), (*C.uint32_t)(unsafe.Pointer(&groupMembers[0])),
		C.size_t(g), (*C.uint32_t)(unsafe.Pointer(&typeNow[0])), (*C.uint8_t)(unsafe.Pointer(&status[0])),
		(*C.uint32_t)(unsafe.Pointer(&first[0]))))
	return typeNow[:n], status[:n], first[:g], err
}

// classifyViable's contract with one resource per vGPU type for the rules of vgpuRules (bit r: rule r); keys is
// vfVgpuTypes' output.  gnuma is filled when topo, blockers when viable (else both nil).  out must be wired and pinned as
// for classifyRules.
func (k *kxpu) classifyVfVgpu(out *C.kxpu_classify_out, rules []C.kxpu_xpu_rule, vgpuRules uint32, recs []C.kxpu_devrec,
	keys []C.kxpu_vgpukey, devRule []uint8, topo, viable bool) (blockers []uint32, gnuma []uint64, err error) {
	n := len(recs)
	if n == 0 {
		return nil, nil, nil
	}
	var np *C.uint64_t
	var bp *C.uint32_t
	if topo {
		gnuma = make([]uint64, n)
		np = (*C.uint64_t)(unsafe.Pointer(&gnuma[0]))
	}
	if viable {
		blockers = make([]uint32, n)
		bp = (*C.uint32_t)(unsafe.Pointer(&blockers[0]))
	}
	var kp *C.kxpu_vgpukey
	if len(keys) > 0 {
		kp = &keys[0]
	}
	rc := C.kxpu_classify_vf_vgpu(k.ctx, &rules[0], C.size_t(len(rules)), C.uint32_t(vgpuRules), &recs[0], C.size_t(n), kp,
		out, (*C.uint8_t)(unsafe.Pointer(&devRule[0])), np, bp)
	if topo {
		gnuma = gnuma[:out.n_groups]
	}
	if viable {
		blockers = blockers[:out.n_groups]
	}
	return blockers, gnuma, kxCheck(k.ctx, "kxpu_classify_vf_vgpu", rc)
}
