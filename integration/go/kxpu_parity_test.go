// kxpu_parity_test.go -- tests to add to pkg/device_plugin of the reference once a Go toolchain is
// available (SURVEY.md section 8(c), last row).  They run the UNMODIFIED reference functions
// against the fixtures of this repository and compare with the values the C oracle produced
// (tests/golden/golden.json, cfg1.yaml, cfg1.json): a green run turns "parity unpinned" into
// "pinned".  NOT compiled here: the build image has no Go toolchain.
//
//	KXPU_REPO=/path/to/this/repo go test ./pkg/device_plugin -run Kxpu
package device_plugin

import (
	"bufio"
	"bytes"
	"compress/gzip"
	"crypto/sha256"
	"encoding/hex"
	"encoding/json"
	"fmt"
	"io"
	"os"
	"path/filepath"
	"strings"
	"testing"

	pluginapi "k8s.io/kubelet/pkg/apis/deviceplugin/v1beta1"
)

type kxGolden struct {
	Rows            int    `json:"rows"`
	DumpSha256      string `json:"dump_sha256"`
	NvidiaRows      int    `json:"nvidia_rows"`
	NvidiaDumpSha256 string `json:"nvidia_dump_sha256"`
}

func kxRepo(t *testing.T) string {
	r := os.Getenv("KXPU_REPO")
	if r == "" {
		t.Skip("KXPU_REPO not set")
	}
	return r
}

// the pci.ids fixture (tests/golden/pci.ids.gz) unpacked into a temp file
func kxPciIds(t *testing.T) string {
	f, err := os.Open(filepath.Join(kxRepo(t), "tests", "golden", "pci.ids.gz"))
	if err != nil {
		t.Fatal(err)
	}
	defer f.Close()
	z, err := gzip.NewReader(f)
	if err != nil {
		t.Fatal(err)
	}
	text, err := io.ReadAll(z)
	if err != nil {
		t.Fatal(err)
	}
	p := filepath.Join(t.TempDir(), "pci.ids")
	if err := os.WriteFile(p, text, 0o644); err != nil {
		t.Fatal(err)
	}
	return p
}

// every NVIDIA device id of the file, in file order (the same enumeration as make_golden.py)
func kxNvidiaIds(t *testing.T, path string) []string {
	f, err := os.Open(path)
	if err != nil {
		t.Fatal(err)
	}
	defer f.Close()
	var ids []string
	seen := map[string]bool{}
	in := false
	sc := bufio.NewScanner(f)
	for sc.Scan() {
		l := sc.Text()
		switch {
		case strings.HasPrefix(l, "10de"):
			in = true
		case in && strings.HasPrefix(l, "\t") && !strings.HasPrefix(l, "\t\t") && len(l) >= 5:
			if !seen[l[1:5]] { // the table holds one row per distinct id (first occurrence)
				seen[l[1:5]] = true
				ids = append(ids, l[1:5])
			}
		case in && !strings.HasPrefix(l, "#") && !strings.HasPrefix(l, "\t"):
			in = false
		}
	}
	return ids
}

// getDeviceName for all 1 859 NVIDIA ids == the oracle's canonical dump
func TestKxpuNvidiaNamesMatchOracle(t *testing.T) {
	pciIdsFilePath = kxPciIds(t)
	raw, err := os.ReadFile(filepath.Join(kxRepo(t), "tests", "golden", "golden.json"))
	if err != nil {
		t.Fatal(err)
	}
	var g kxGolden
	if err := json.Unmarshal(raw, &g); err != nil {
		t.Fatal(err)
	}
	var dump bytes.Buffer
	ids := kxNvidiaIds(t, pciIdsFilePath)
	for _, id := range ids {
		fmt.Fprintf(&dump, "10de:%s\t%s\n", id, getDeviceName(id))
	}
	if len(ids) != g.NvidiaRows {
		t.Fatalf("nvidia ids: got %d want %d", len(ids), g.NvidiaRows)
	}
	sum := sha256.Sum256(dump.Bytes())
	if hex.EncodeToString(sum[:]) != g.NvidiaDumpSha256 {
		t.Fatalf("canonical dump differs from the oracle's (sha256 %s)", hex.EncodeToString(sum[:]))
	}
}

// cfg1 of SURVEY 8(d): one H100 in group 214 -> maps, resource name, CDI YAML
func TestKxpuCfg1(t *testing.T) {
	pciIdsFilePath = kxPciIds(t)
	root := t.TempDir()
	// entries of /sys/bus/pci/devices are symlinks: filepath.Walk lstat()s them, so they are "not a directory"
	real := filepath.Join(root, "real", "0000:c1:00.0")
	os.MkdirAll(real, 0o755)
	os.WriteFile(filepath.Join(real, "vendor"), []byte("0x10de\n"), 0o644)
	os.WriteFile(filepath.Join(real, "device"), []byte("0x2330\n"), 0o644)
	os.Symlink("../../../bus/pci/drivers/vfio-pci", filepath.Join(real, "driver"))
	os.Symlink("../../../kernel/iommu_groups/214", filepath.Join(real, "iommu_group"))
	base := filepath.Join(root, "devices")
	os.MkdirAll(base, 0o755)
	os.Symlink(real, filepath.Join(base, "0000:c1:00.0"))
	basePath = base

	createIommuDeviceMap()
	if len(iommuMap) != 1 || len(iommuMap["214"]) != 1 || iommuMap["214"][0].addr != "0000:c1:00.0" || iommuMap["214"][0].index != 0 {
		t.Fatalf("iommuMap = %v", iommuMap)
	}
	if len(deviceMap) != 1 || len(deviceMap["2330"]) != 1 || deviceMap["2330"][0] != "214" {
		t.Fatalf("deviceMap = %v", deviceMap)
	}
	if n := getDeviceName("2330"); n != "GH100_H100_SXM5_80GB" {
		t.Fatalf("getDeviceName(2330) = %q", n)
	}
	// generateCDISpec writes cdiConfigPath + "cdi-vfio-xxxx.yaml"; compare with tests/golden/cfg1.yaml
	// (cdiConfigPath is a constant in the reference: run this test where /var/run/cdi is writable,
	// or make it a variable like the other seams)
	generateCDISpec(iommuMap)
	got, err := os.ReadFile("/var/run/cdi/cdi-vfio-xxxx.yaml")
	if err != nil {
		t.Skip("cannot read the CDI file back: ", err)
	}
	want, _ := os.ReadFile(filepath.Join(kxRepo(t), "tests", "golden", "cfg1.yaml"))
	if !bytes.Equal(got, want) {
		t.Fatalf("CDI YAML differs from the oracle's:\n%s\n--- want\n%s", got, want)
	}
}

// kxpu_lw_encode_topo: the ListAndWatchResponse with Device.topology that gogo's Marshal (kubelet v0.30 api.pb.go:
// fields in number order, a zero int64 skipped) produces, against the oracle's bytes for the same list.
func TestKxpuListAndWatchTopology(t *testing.T) {
	node := func(ids ...int64) *pluginapi.TopologyInfo {
		ti := &pluginapi.TopologyInfo{}
		for _, id := range ids {
			ti.Nodes = append(ti.Nodes, &pluginapi.NUMANode{ID: id})
		}
		return ti
	}
	resp := &pluginapi.ListAndWatchResponse{Devices: []*pluginapi.Device{
		{ID: "214", Health: pluginapi.Healthy, Topology: node(0, 1)},
		{ID: "7", Health: pluginapi.Unhealthy},
		{ID: "30", Health: pluginapi.Healthy, Topology: node(63)},
	}}
	got, err := resp.Marshal()
	if err != nil {
		t.Fatal(err)
	}
	// oracle/kxpu_topo_oracle.c: kxo_lw_encode_topo([214, 7, 30], [1, 0, 1], [0b11, 0, 1 << 63])
	want := "0a160a0332313412074865616c7468791a060a000a0208010a0e0a01371209556e6865616c7468790a130a02333012074865616c7468791a040a02083f"
	if hex.EncodeToString(got) != want {
		t.Fatalf("topology wire bytes differ:\n got %x\nwant %s", got, want)
	}
}

// kxpu_preferred_allocation_pcie on the worked example of include/kxpu.h (tests/pcie_example.py): two sockets, a host
// bridge each with two root ports, a switch under each root port and two GPUs under each switch; groups 10-13 on NUMA
// node 0, 20-23 on node 1, positions 0..7.  The answers are the C oracle's (oracle/kxpu_pcie_oracle.c).
func TestKxpuPreferredAllocationPcie(t *testing.T) {
	k, err := newKxpu(0)
	if err != nil {
		t.Skip(err)
	}
	var bdfs, targets []string
	for _, hb := range []int{0x00, 0x80} {
		// root port, switch, down port, GPU (bus offsets from the host bridge's bus)
		ports := [][4]string{{"%02x:01.0", "%02x:00.0", "%02x:00.0", "%02x:00.0"}, {"%02x:01.0", "%02x:00.0", "%02x:01.0", "%02x:00.0"},
			{"%02x:02.0", "%02x:00.0", "%02x:00.0", "%02x:00.0"}, {"%02x:02.0", "%02x:00.0", "%02x:01.0", "%02x:00.0"}}
		buses := [][4]int{{0, 1, 2, 3}, {0, 1, 2, 4}, {0, 5, 6, 7}, {0, 5, 6, 8}}
		for i, r := range ports {
			var c [4]string
			for j := range r {
				c[j] = fmt.Sprintf(r[j], hb+buses[i][j])
			}
			bdf := "0000:" + c[3]
			bdfs = append(bdfs, bdf)
			targets = append(targets, fmt.Sprintf("../../../devices/pci0000:%02x/0000:%s/0000:%s/0000:%s/%s", hb, c[0], c[1], c[2], bdf))
		}
	}
	nodes, parent, depth, err := k.pcieTreeOfLinks(bdfs, targets, []uint32{0, 1, 2, 3, 4, 5, 6, 7, 8}, []uint32{0, 1, 2, 3, 4, 5, 6, 7})
	if err != nil || len(parent) != 18 {
		t.Fatalf("pcieTree: %v, %d nodes", err, len(parent))
	}
	masks := []uint64{1, 1, 1, 1, 2, 2, 2, 2}
	all := []uint32{0, 1, 2, 3, 4, 5, 6, 7}
	but := func(x uint32) []uint32 {
		var r []uint32
		for _, p := range all {
			if p != x {
				r = append(r, p)
			}
		}
		return r
	}
	avail := [][]uint32{all, but(0), but(0), but(2), all, all}
	must := [][]uint32{nil, nil, nil, nil, {2}, nil}
	size := []uint32{2, 2, 1, 1, 3, 5}
	want := [][]uint32{{0, 1}, {2, 3}, {1}, {3}, {2, 3, 0}, {0, 1, 2, 3, 4}}
	got, err := k.preferredAllocationPcie(masks, nodes, parent, depth, avail, must, size)
	if err != nil || fmt.Sprint(got) != fmt.Sprint(want) {
		t.Fatalf("preferredAllocationPcie: %v %v, want %v", got, err, want)
	}
}
