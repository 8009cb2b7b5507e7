// device_plugin.hpp -- host side of the discovery hot path, above the C ABI (include/kxpu.h).
//
// The reference host is Go; this image has no Go toolchain, so the host logic that sits
// above libkxpu.so is written in C++ and mirrors the reference's package
// pkg/device_plugin one to one: same function names, same package-level seams
// (basePath, pciIdsFilePath, readLink, readIDFromFile -- device_plugin.go:36-39,
// returnIommuMap -- generic_device_plugin.go:34), same argument meaning, same error
// behaviour ("log and degrade": unreadable entries are skipped, an unknown device id
// falls back to the raw id, an Allocate re-validation failure is an error naming the bdf).
// The syscalls (walk, read, readlink) stay on the host exactly where the reference does
// them; everything per-device / per-byte after that goes through the kxpu_* calls.
// The gRPC server itself (Register / ListAndWatch stream / Allocate handler plumbing,
// generic_device_plugin.go:128-220) is out of scope and stays in the Go binary; the Go
// cgo shim that replaces this file in production is shown in INTEGRATION.md.
#pragma once
#include <atomic>
#include <cstdint>
#include <deque>
#include <functional>
#include <map>
#include <optional>
#include <set>
#include <shared_mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/kxpu.h"

namespace device_plugin {

// pkg/device_plugin/device_plugin.go:24-28
struct NvidiaGpuDevice {
    std::string addr;    // PCI address of device
    uint64_t index;      // PCI device index on PCI bus
    size_t xpuClass = 0; // index into Plugin::xpuClasses of the class this function matched
    int64_t cdev = -1;   // N of its VFIO cdev /dev/vfio/devices/vfio<N> (XpuClass::vfioCdev only); -1 = none
    uint32_t vgpuType = 0;  // XpuClass::vfVgpu only: the vGPU type ID the walk read from nvidia/current_vgpu_type
    std::string vgpuKey{};  // XpuClass::vfVgpu only: that type's key, the name of the plugin that serves the VF
};

// One mediated device (vGPU) of the mdev walk: the mdevMap counterpart of NvidiaGpuDevice
struct MdevDevice {
    std::string uuid;      // entry name under mdevBasePath
    std::string parent;    // PCI address of the parent device
    uint64_t index;        // busIndex of the mdev walk
    size_t vgpuClass = 0;  // index into Plugin::vgpuClasses of the class this mdev matched
    int64_t cdev = -1;     // N of its VFIO cdev /dev/vfio/devices/vfio<N> (XpuClass::mdevCdev only); -1 = none
};

// Go maps iterate in random order; the canonical order used here (and by the oracle) is
// first-seen walk order, which is one of the orders the reference can produce.
template <typename V>
using OrderedMap = std::vector<std::pair<std::string, V>>;

// pkg/device_plugin/generic_device_plugin.go:35-48 (the fields the hot path touches)
struct Device {  // pluginapi.Device
    std::string ID;
    std::string Health;
    uint64_t numa = 0;  // Device.Topology: bit k = NUMA node k (the group's mask); 0 = no topology
    // the group's node in Plugin::pcieParent / pcieDepth (pcieTopologyAware); a vGPU plugin's device: in
    // Plugin::mdevPcieParent / mdevPcieDepth (vgpuPcieTopologyAware)
    uint32_t pcieNode = KXPU_PCIE_NO_NODE;
    // groupViability: why VFIO cannot open the group ("<bdf> is bound to <driver>"), from the last walk; empty = viable.
    // Separate from Health, which the HealthWatcher flips: the device is sent Unhealthy when either says so.
    std::string blocker{};
    // aerHealth: why the group's PCIe AER counters are over a limit ("<bdf> reported <n> fatal uncorrectable PCIe errors
    // (limit <l>)"), from the last walk or refreshAerHealth; empty = within the limits.  Also sent Unhealthy.
    std::string aer{};
    // vfVgpuHealth: why the VF's vGPU type is no longer the one the walk saw ("<vf> now carries vGPU type 0 (was 557)"),
    // from the last refreshVfVgpuTypes; empty = unchanged, and after every rediscover.  Also sent Unhealthy.
    std::string drift{};
    // a plugin of a class with XpuClass::resourceNames: the model name of the group (the pci.ids name of its first
    // member's device id, else that raw id), which ResourceSlices publishes as productName; empty elsewhere, where the
    // plugin's devpluginName is that name
    std::string model{};
};
// pluginapi.DevicePluginOptions (GetDevicePluginOptions, generic_device_plugin.go:253-258)
struct DevicePluginOptions {
    bool PreStartRequired = false;
    bool GetPreferredAllocationAvailable = false;
};
// pluginapi.ContainerPreferredAllocationRequest / ContainerPreferredAllocationResponse
struct ContainerPreferredAllocationRequest {
    std::vector<std::string> AvailableDeviceIDs;
    std::vector<std::string> MustIncludeDeviceIDs;
    int32_t AllocationSize = 0;
};
struct ContainerPreferredAllocationResponse {
    std::vector<std::string> DeviceIDs;
};
struct GenericDevicePlugin {
    std::string devpluginName;   // resource name suffix: "<resourceNamespace>/<devpluginName>" (:211)
    std::string resourceNamespace = "nvidia.com";  // DevicePluginNamespace (:26), per class (XpuClass)
    size_t xpuClass = 0;         // index into Plugin::xpuClasses (Plugin::vgpuClasses when vgpu)
    bool vgpu = false;           // serves one vGPU type (devs are mdev IOMMU groups)
    std::string socketPath;      // DevicePluginPath + "kata-xpu-<name>.sock" (:76)
    std::string devicePath;      // "/dev/vfio/" (device_plugin.go:105)
    std::vector<Device> devs;
    std::string deviceKey;       // the device id (passthrough) or type key (vgpu) the plugin serves; matches it on rediscovery
    // XpuClass::vfioCdev only: device ID -> the node names under devicePath the health watcher watches (one per member,
    // "vfio<N>"); an ID not listed is watched as devicePath/<ID>
    std::map<std::string, std::vector<std::string>> nodes;
};

// pluginapi.ContainerAllocateResponse as Allocate fills it (generic_device_plugin.go:304-350)
struct ContainerAllocateResponse {
    std::map<std::string, std::string> Envs;
    std::vector<std::string> CDIDevices;  // CDIDevice{Name}
};

struct Error {
    bool failed = false;
    std::string message;
    explicit operator bool() const { return failed; }
};

// healthCheck (generic_device_plugin.go:389-457) + the re-send half of ListAndWatch (:222-250) for
// ONE plugin: an inotify watch on devicePath/<ID> of every device; Remove / Rename of the path marks
// the device Unhealthy, Create marks it Healthy.  The reference sends one ListAndWatchResponse per
// event; here poll() drains the whole queue, flips Health of the matching devs and reports how many
// changed, and the caller re-encodes the list ONCE per batch (Plugin::ListAndWatchBytes): the last
// response of a burst is byte-identical to the reference's last response.
// watchCreates = false mirrors the reference exactly: it only adds the device paths themselves (and the
// directory of the kubelet socket, which is out of scope here), so a Create of /dev/vfio/<group> is
// never seen.  watchCreates = true also watches devicePath itself, which is what the code intends.
class HealthWatcher {
  public:
    HealthWatcher(GenericDevicePlugin &dp, bool watchCreates = false);
    ~HealthWatcher();
    HealthWatcher(const HealthWatcher &) = delete;
    HealthWatcher &operator=(const HealthWatcher &) = delete;
    Error start();             // watcher.Add(devicePath/ID) for every dev (:421-430)
    // after a rediscovery changed the plugin's device list: watch the IDs that are new, drop the watches of IDs that left
    Error resync();
    int poll(int timeout_ms);  // #devs whose Health changed in this batch; 0 = none; -1 = error
    uint64_t events() const { return events_; }

  private:
    GenericDevicePlugin &dp_;
    bool watchCreates_;
    int fd_ = -1, dirWd_ = -1;
    std::map<int, std::string> wdToId_;
    std::map<int, std::string> wdToNode_;  // the node name each watch is on
    std::vector<std::string> nodesOf(const std::string &id) const;
    uint64_t events_ = 0;
    int setHealth(const std::string &id, const char *health);
};

// SURVEY 8(f) row 2, second half: what makes a snapshot of the discovery trustworthy.  Allocate
// re-validates every device against sysfs (readlink iommu_group + read vendor, two syscalls per device,
// generic_device_plugin.go:329-338) because a device may have been re-bound since discovery.  The kernel
// announces exactly that: bind / unbind / add / remove uevents of the pci subsystem on the
// NETLINK_KOBJECT_UEVENT socket (bind / unbind since Linux 4.14).  BindWatcher counts them: while the
// generation it reports equals the one recorded at discovery, no PCI function changed its driver and the
// snapshot answers what the live reads would answer.
class BindWatcher {
  public:
    BindWatcher() = default;
    ~BindWatcher();
    BindWatcher(const BindWatcher &) = delete;
    BindWatcher &operator=(const BindWatcher &) = delete;
    Error start();            // opens the uevent socket (needs no privilege beyond a netlink socket)
    bool healthy() const { return fd_ >= 0 && !lost_; }
    // drains the socket; the generation grows by one per pci bind / unbind / add / remove event and jumps
    // when the kernel reports lost messages (ENOBUFS): then nothing can be said about what was missed
    uint64_t generation();
    // a separate counter for the mdev bus: grows by one per mdev add / remove / bind / unbind event (a vGPU created or
    // destroyed), and jumps with generation() on lost messages.  generation() never counts mdev events, so the PCI
    // snapshot of Allocate stays valid while vGPUs come and go.  Drains the socket like generation().
    uint64_t mdevGeneration();
    // feeds one raw uevent message (tests; also what generation() calls per datagram)
    void feed(const char *msg, size_t len);

  private:
    int fd_ = -1;
    bool lost_ = false;
    uint64_t gen_ = 0, mdevGen_ = 0;
};

// One kind of accelerator the plugin serves (the reference hard-codes the NVIDIA one: nvidiaVendorID
// device_plugin.go:19, the vfio-pci check :156, DevicePluginNamespace / CdiVendorClass
// generic_device_plugin.go:26,31, the CDI file name device_plugin.go:79).
struct XpuClass {
    std::string vendor;             // vendor id as readIDFromFile returns it, e.g. "1002"
    std::string driver;             // basename of the driver link, e.g. "vfio-pci"
    std::string resourceNamespace;  // resource = <resourceNamespace>/<device name>
    std::string cdiKind;            // CDI kind of this class's spec file and Allocate names
    std::string cdiFileStem;        // <cdiConfigPath><cdiFileStem>.yaml|.json
    // DRA driver name that publishes this class's IOMMU groups as ResourceSlices (Plugin::ResourceSlices, or
    // Plugin::VgpuResourceSlices for a vGPU class); empty: the class is not published
    std::string draDriver{};
    // passthrough only (a vGPU class with it is refused): the class's functions are reached through their VFIO cdevs.  The
    // gathers read <bdf>/vfio-dev/ of every function that matches the class, the CDI spec names /dev/vfio/devices/vfio<N>
    // (kxpu_cdi_emit_cdev), the health watcher watches those nodes, and a group with a member without a cdev is treated
    // like a group that is not viable.  false: nothing under vfio-dev/ is opened and every output is as without it.
    bool vfioCdev = false;
    // vGPU only (a passthrough class with it is refused): the class's mdevs are reached through their VFIO cdevs.  The mdev
    // walk reads <uuid>/vfio-dev/ of every mdev that matches the class, the CDI spec names /dev/vfio/devices/vfio<N>
    // (kxpu_cdi_emit_mdev_cdev), the health watcher watches those nodes, and a group whose mdev has no cdev is withheld
    // like a passthrough group that is not viable.  Kept apart from vfioCdev because it also rests on the vGPU driver
    // registering a cdev.  false: nothing under vfio-dev/ is opened and every output is as without it.
    bool mdevCdev = false;
    // passthrough only (refused on a vGPU class and together with draDriver): the class serves vGPUs that live on SR-IOV
    // virtual functions (include/kxpu.h, kxpu_vf_vgpu_types).  For every VF of the class (a record with a physfn link) the
    // PCI walk reads nvidia/current_vgpu_type and nvidia/creatable_vgpu_types; the class gets one plugin per vGPU type
    // key, <resourceNamespace>/<type key>, with no pci.ids lookup, and a VF that carries no type (the PF, a free VF) is
    // never offered.  false: nothing under nvidia/ is opened and every output is as without it.
    bool vfVgpu = false;
    // vfVgpu only: type ID -> name, the first name table of kxpu_vf_vgpu_types.  A restart on a GPU whose VFs are all taken
    // finds no creatable_vgpu_types list to learn names from; with Plugin::resumeIndices the class's spec carries the type
    // of every VF it names, and the restart learns the names from it, so these are needed only without resumeIndices.
    std::map<uint32_t, std::string> vgpuTypeNames{};
    // vfVgpu only (refused on any other class): the DRA driver that publishes the class's vGPUs as ResourceSlices
    // (Plugin::VfVgpuResourceSlices, kxpu_dra_slices_vf_vgpu), one pool named nodeName.  Kept apart from draDriver, which
    // promises the passthrough record layout (kxpu_dradev).  Empty: the class's vGPUs are not published.
    std::string vgpuDraDriver{};
    // passthrough only (refused on a vfVgpu class and on a vGPU class): device id -> resource name, replacing the pci.ids
    // name (include/kxpu.h, kxpu_classify_named).  A key is a device id exactly as readIDFromFile returns it ("2330"),
    // or "*" for every other device id of the class; a value is a Kubernetes qualified name.  {"*": "pgpu"} serves
    // every device of the class as <resourceNamespace>/pgpu.  The class's entries whose final names are equal -- two ids
    // with one configured name, or two unlisted ids with one pci.ids name -- are served by one plugin, groups in walk
    // order, whose deviceKey is that name.  Empty (default): the class is named and split per device id as above.
    std::map<std::string, std::string> resourceNames{};
};
XpuClass defaultXpuClass();  // {"10de", "vfio-pci", "nvidia.com", "nvidia.com/gpu", "cdi-vfio-xxxx"}

// What Plugin::rediscover changed.  Positions are indices into Plugin::devicePlugins.
struct RediscoverReport {
    std::vector<size_t> changedPlugins;  // device list changed: re-send ListAndWatch, resync the health watcher
    std::vector<size_t> addedPlugins;    // new resources: Start and Register them (then they count as changed too)
    kxpu_reconcile_counts pci{}, mdev{}; // kept / new / changed / retired of each walk, and its next index
    std::vector<std::string> cdiFilesWritten;  // spec files whose bytes changed (rewritten atomically)
};

// What Plugin::resumeIndices did at start-up for one walk (PCI or mdev).
struct ResumeWalk {
    kxpu_reconcile_counts counts{};      // the previous specs' entries against the first walk, and the next index
    std::vector<std::string> filesRead;  // spec files read and parsed (a missing file is not listed)
    std::string fallback;                // why the walk resumed from nothing known; empty: it resumed from its specs
    std::set<size_t> typedClasses;       // vfVgpu classes whose spec was read in a typed layout (each VF's vGPU type)
};
struct ResumeReport {
    ResumeWalk pci, mdev;
    bool stateRead = false;                    // the index state file was there and well formed
    uint64_t statePci = 0, stateMdev = 0;      // its values (0 when it was not read)
    std::vector<std::string> filesWritten;     // spec and state files whose bytes changed at start-up
};

// The length of a label string Plugin::MetricsText keeps: len up to KXPU_METRICS_STRING_MAX, else that limit, moved back
// to the lead of a UTF-8 sequence the limit would split (exposed for CPU tests)
size_t metricsCut(const uint8_t *s, size_t len);
// the atomic spec writer of Plugin::rediscover (exposed for CPU tests)
Error writeSpecFileAtomicForTests(const std::string &file_path, const uint8_t *doc, size_t len, bool &written);
// The index state file of Plugin::resumeIndices: "pci <next>\nmdev <next>\n", canonical decimals.  format / parse are
// exact inverses; parse refuses anything else.
std::string formatIndexState(uint64_t pciNext, uint64_t mdevNext);
bool parseIndexState(const std::string &text, uint64_t &pciNext, uint64_t &mdevNext);

// The output arrays of one classify call (kxpu_classify_out + dev_rule + group_numa) and their counts.
struct ClassifyResult {
    std::vector<uint32_t> accept, gids, goff, gmem, doff, dgrp;
    std::vector<uint64_t> dids, gnuma;
    std::vector<uint32_t> gblk;  // groupViability: first blocking record per group ordinal, or KXPU_VIABLE
    std::vector<uint8_t> drule;
    std::vector<uint32_t> dslot;  // some class has resourceNames: the slot of every deviceMap entry, or KXPU_NO_SLOT
    uint32_t nGroups = 0, nDevids = 0;
    // sizes the arrays for n records and points a kxpu_classify_out at them
    kxpu_classify_out wire(size_t n);
};

// One walk's classify result, kept so that the maps can be rebuilt with reconciled indices (host bookkeeping).
struct PciWalk {
    std::vector<kxpu_devrec> recs;
    ClassifyResult out;
    // pcieTopologyAware: the path of every record and the walk's PCIe forest (kxpu_pcie_tree)
    std::vector<kxpu_pcipath> paths;
    std::vector<uint32_t> gnode, nodeParent;
    std::vector<uint64_t> nodeKey;
    std::vector<uint8_t> nodeDepth;
    uint32_t nNodes = 0;
    // some class has vfioCdev: per record, N of its VFIO cdev, -1 = none or not read
    std::vector<int64_t> cdevs;
    // sriovAware: per record its physfn / sriov_numvfs reads, and kxpu_sriov's pf_of and numvfs; per group ordinal the
    // first blocking member or KXPU_VIABLE
    std::vector<kxpu_sriovrec> srs;
    std::vector<uint32_t> pfOf, numvfs, gsriov;
    // draPcieDomain: per group ordinal its root port and switch (kxpu_pcie_ports), or KXPU_PCIE_NO_KEY
    std::vector<uint64_t> rootPort, pcieSwitch;
    // aerPortHealth: kxpu_aer_ports' CSR, the ports above every record (aerPortOf[aerPortOff[i] .. aerPortOff[i+1]),
    // nearest first), and each port's function key
    std::vector<uint32_t> aerPortOff, aerPortOf;
    std::vector<uint64_t> aerPortKey;
    // resetCheck: per record its reset_method (or reset) read, and kxpu_reset_check's methods and set verdict; per group
    // ordinal the reset blocker or KXPU_VIABLE
    std::vector<kxpu_resetrec> rrs;
    std::vector<uint8_t> rmeth;
    std::vector<uint32_t> rset, greset;
    // some class has vfVgpu: per record its current_vgpu_type read and creatable_vgpu_types text, and kxpu_vf_vgpu_types'
    // key row, type ID and status
    std::vector<kxpu_vfvgpurec> vts;
    std::vector<std::string> creatable;
    std::vector<kxpu_vgpukey> vkeys;
    std::vector<uint32_t> vtype;
    std::vector<uint8_t> vstatus;
    // vfVgpuDraEnabled or vfVgpuHealth only, one per record of vts: the basename of its physfn link (the PF's address);
    // "" = not read
    std::vector<std::string> physfn;
};
struct MdevWalk {
    std::vector<kxpu_mdevrec> recs;
    ClassifyResult out;
    std::vector<uint32_t> koff;
    std::vector<uint8_t> keys;
    // vgpuDraEnabled only, one per record: the parent's device id (<uuid>/../device) and the PCIe root of the entry's
    // link; "" = not read, failed or outside kxpu_dramdev's domain
    std::vector<std::string> parentDevice, pcieRoot;
    // readsMdevPaths, one per record: the entry's link as a kxpu_pcipath (len 0: not read or unknown); with
    // vgpuPcieTopologyAware, the walk's PCIe forest (kxpu_pcie_tree_mdev)
    std::vector<kxpu_pcipath> paths;
    std::vector<uint32_t> gnode, nodeParent;
    std::vector<uint64_t> nodeKey;
    std::vector<uint8_t> nodeDepth;
    uint32_t nNodes = 0;
    // draVgpuPcie (with a vGPU class that has a draDriver): per group ordinal its root port and switch
    // (kxpu_pcie_ports_mdev), or KXPU_PCIE_NO_KEY
    std::vector<uint64_t> rootPort, pcieSwitch;
    // aerPortHealth: kxpu_aer_ports_mdev's CSR and keys, the ports above every mdev's parent, as in PciWalk
    std::vector<uint32_t> aerPortOff, aerPortOf;
    std::vector<uint64_t> aerPortKey;
    // mdevCdevEnabled only, one per record: N of its VFIO cdev, -1 = none or not read
    std::vector<int64_t> cdevs;
    // vgpuSriovAware only, one per record: its physfn read (kxpu_sriovrec, physfn only) and kxpu_mdev_pf's answer, the
    // PF's index in the PCI walk's records or KXPU_NO_PF
    std::vector<kxpu_sriovrec> srs;
    std::vector<uint32_t> pfOf;
};

// The host state of one IOMMU group of a walk (Plugin::iommuState / mdevState, same positions as iommuMap / mdevMap).
// A field whose setting is off keeps its default.
template <typename Dra>  // kxpu_dradev (passthrough) or kxpu_dramdev (vGPU)
struct GroupState {
    size_t klass = 0;  // index into xpuClasses (vgpuClasses): the class of the group's first member
    uint64_t numa = 0;  // topologyAware: the group's NUMA mask; 0 = no topology
    // pcieTopologyAware: the group's node in pcieParent / pcieDepth; a vGPU group (vgpuPcieTopologyAware): in
    // mdevPcieParent / mdevPcieDepth
    uint32_t pcieNode = KXPU_PCIE_NO_NODE;
    // why VFIO cannot open the group, empty = it can: "<bdf> is bound to <driver>" (groupViability), else "<bdf> has no
    // VFIO cdev" (vfioCdev), else sriov; a vGPU group: "<uuid> has no VFIO cdev" (mdevCdev)
    std::string blocker{};
    // the check that produced blocker (KXPU_MR_NOT_VIABLE, _VFIO_CDEV_MISSING, _SRIOV or _RESET); read only while blocker
    // is not empty.  The metrics name the reason by it (Plugin::MetricsText)
    uint32_t blockerKind = KXPU_MR_NOT_VIABLE;
    std::string sriov{};  // sriovAware, passthrough only: the SR-IOV reason; empty = served
    std::string reset{};  // resetCheck, passthrough only: why a member cannot be reset between tenants; empty = served
    std::string aer{};    // aerHealth: the first member over an AER limit (computeAer); empty = within the limits
    uint8_t aerBits = 0;  // aerHealth: the group's KXPU_AER_* bits (computeAer)
    // aerHealth: the highest known TOTAL_ERR_FATAL / _NONFATAL over the files computeAer folded for the group (members, an
    // mdev's parent, a VF's PF); KXPU_METRICS_NO_VALUE = none known.  Reported by MetricsText only
    uint64_t aerMax[2] = {KXPU_METRICS_NO_VALUE, KXPU_METRICS_NO_VALUE};
    // aerPortHealth: the PCIe ports above the group's members (kxpu_aer_ports[_mdev]), member by member, each nearest
    // first and each port once: (port address, the function it was found above: a member, or an mdev's parent)
    std::vector<std::pair<std::string, std::string>> aerPorts{};
    std::optional<Dra> dra{};  // draEnabled (vgpuDraEnabled): the ResourceSlice record of its first member; none = unpublished
    // vfVgpuDraEnabled, a group of a class with a vgpuDraDriver whose first member is a VF that carries a named vGPU type:
    // its VF-vGPU ResourceSlice record; none = unpublished
    std::optional<kxpu_dravfvgpu> vfVgpuDra{};
    // vfVgpuHealth, a group of a vfVgpu class whose first member is a VF: the PF's address (its physfn basename);
    // sriovPfAware, a group of another passthrough class whose first member is a VF of a PF in the walk (kxpu_sriov's
    // pf_of): that PF's address; vgpuSriovAware, a vGPU group whose first mdev's parent is a VF of a PF in the PCI walk:
    // that PF's address
    std::string pf{};
    // vgpuSriovAware and vgpuDraEnabled, a vGPU group with a pf: the PF's device id and model name (getDeviceNames);
    // sriovPfAware and draEnabled, a passthrough group with a pf: the PF's device id (pfProduct stays empty); "" = not
    // known
    std::string pfDevice{}, pfProduct{};
    // vfVgpuHealth: the drift reason of the group's first member (Device::drift); empty = its type is the walk's
    std::string drift{};
    // passthrough: the device id of the group's first member (readIDFromFile's text); names Device::model
    std::string firstDevice{};
    // draPcieDomain, PCI walk: the group's root port and nearest switch upstream port (kxpu_pcie_ports' function keys),
    // or KXPU_PCIE_NO_KEY; draVgpuPcie, mdev walk: the same keys of the group's parent GPU (kxpu_pcie_ports_mdev)
    uint64_t rootPort = KXPU_PCIE_NO_KEY, pcieSwitch = KXPU_PCIE_NO_KEY;
};

class Plugin {
  public:
    // ---- seams (device_plugin.go:36-39, generic_device_plugin.go:34)
    std::string basePath = "/sys/bus/pci/devices";
    std::string pciIdsFilePath = "/usr/pci.ids";
    std::string cdiConfigPath = "/var/run/cdi/";  // device_plugin.go:20
    std::function<bool(const std::string &base, const std::string &addr, const std::string &link, std::string &out)> readLink;
    std::function<bool(const std::string &base, const std::string &addr, const std::string &prop, std::string &out)> readIDFromFile;
    std::function<const OrderedMap<std::vector<NvidiaGpuDevice>> &()> returnIommuMap;
    // Allocate re-validation (generic_device_plugin.go:329-338).  false (default) = the reference's live
    // reads for every device of every request.  true = answer from the discovery snapshot as long as
    // bindGeneration() still returns the value recorded by createIommuDeviceMap; any change (or an
    // unhealthy watcher) falls back to the live reads for that request.  bindGeneration is a seam: by
    // default it asks the BindWatcher (started on first use), tests replace it.
    bool snapshotValidation = false;
    // The accelerator classes served.  Every list, the default (one NVIDIA class) included, goes through
    // kxpu_classify_rules / kxpu_cdi_emit_kind / kxpu_alloc_names_kind; with the default list these return the bytes
    // of the reference's NVIDIA-only calls (include/kxpu.h).  Classes must be distinct (vendor, driver) pairs, at most
    // KXPU_MAX_RULES.  Socket names stay kata-xpu-<name>.sock, so two classes whose devices get the same name collide
    // like two NVIDIA device ids with the same name do in the reference (generic_device_plugin.go:76); only a class
    // with XpuClass::resourceNames resolves that, for its own devices.
    std::vector<XpuClass> xpuClasses{defaultXpuClass()};
    // vGPU classes: mediated devices under mdevBasePath, one resource <resourceNamespace>/<type key> per (class, type
    // key).  vendor = the parent PCI device's vendor id, driver = the mdev's driver.  Empty (default): nothing under
    // mdevBasePath is read and every flow is the one above.  A class's cdiKind and cdiFileStem must differ from those
    // of every other class (xpuClasses and vgpuClasses), else InitiateDevicePlugin fails.
    std::vector<XpuClass> vgpuClasses;
    std::string mdevBasePath = "/sys/bus/mdev/devices";
    std::function<const OrderedMap<std::vector<MdevDevice>> &()> returnMdevMap;
    std::function<bool(uint64_t &generation)> bindGeneration;
    // the mdev counterpart (BindWatcher::mdevGeneration by default); read before each mdev walk
    std::function<bool(uint64_t &generation)> mdevGeneration;
    // NUMA topology (include/kxpu.h, ABI v5).  false (default): nothing named numa_node is opened, the records, the
    // ListAndWatch bytes and the options are the reference's, GetPreferredAllocation answers nothing.  true: the gathers
    // read <entry>/numa_node through readNumaNode (an mdev: its parent's, entry "<uuid>/.."), classify returns a NUMA
    // mask per group, every Device carries its group's mask (ListAndWatch sends Device.topology), and
    // GetPreferredAllocation keeps an allocation on as few nodes as it can (kxpu_preferred_allocation).
    bool topologyAware = false;
    std::function<bool(const std::string &base, const std::string &entry, std::string &out)> readNumaNode;
    // PCIe topology (include/kxpu.h, ABI v7).  false (default): nothing more is read and every output is as above.  true:
    // the PCI gathers read the link <basePath>/<entry> through readPciPath (the whole target), each record keeps its path
    // from the first component that begins with "pci", kxpu_pcie_tree builds the walk's forest, every passthrough Device
    // carries its group's node, and GetPreferredAllocation keeps an allocation under as few PCIe switches as it can
    // (kxpu_preferred_allocation_pcie; vGPU plugins keep the NUMA answer unless vgpuPcieTopologyAware is on).  Both
    // settings may be on together.
    bool pcieTopologyAware = false;
    std::function<bool(const std::string &base, const std::string &entry, std::string &target)> readPciPath;
    // PCIe topology of vGPUs (include/kxpu.h, kxpu_pcie_tree_mdev).  false (default): nothing more is read and every
    // output is as above, the NUMA answer of vGPU plugins under pcieTopologyAware included.  true: the mdev walk reads the
    // link <mdevBasePath>/<uuid> of every entry that got as far as its iommu_group link (readPciPath, the read
    // vgpuDraEnabled does), kxpu_pcie_tree_mdev builds the walk's forest with each mdev below its parent function, every
    // vGPU Device carries its group's node, and GetPreferredAllocation of a vGPU plugin keeps an allocation under as few
    // GPUs, then switches, as it can (kxpu_preferred_allocation_pcie).  It rests on the vGPU manager accepting several
    // vGPUs of one GPU in one VM [assumed], which is why it is a setting of its own.
    bool vgpuPcieTopologyAware = false;
    // IOMMU group viability (include/kxpu.h, ABI v8).  false (default): nothing more is read and every output is as
    // above.  true: for every non-directory entry that is not a class candidate the gathers read its `driver` link (when
    // not read yet); a bound driver that is neither in viabilityDrivers nor the driver of a class makes the entry a
    // blocker of the group its `iommu_group` link names (KXPU_REC_BLOCKS).  Classify runs kxpu_classify_viable; every
    // device of a group with a blocker is sent Unhealthy and Allocate refuses it, naming the blocking function.  CDI specs
    // and vGPU plugins do not change.
    bool groupViability = false;
    std::vector<std::string> viabilityDrivers{"vfio-pci", "pci-stub", "pcieport"};
    // DRA ResourceSlices (include/kxpu.h, ABI v9).  With no XpuClass::draDriver set (default) nothing more is read and
    // every output is as above.  With one: the PCI gathers read numa_node and the entry link as topologyAware /
    // pcieTopologyAware do (none of those settings' other effects turn on), and ResourceSlices publishes the class's
    // groups in one pool named nodeName.  nodeName is a seam: the Go host takes it from NODE_NAME.
    std::string nodeName;
    bool draEnabled() const;  // some class has a draDriver
    // the PCI gathers read numa_node (topologyAware, draEnabled or vfVgpuDraEnabled) and the entry link
    // (pcieTopologyAware, draEnabled, vfVgpuDraEnabled, resetCheck or aerPortHealth)
    bool readsNuma() const { return topologyAware || draEnabled() || vfVgpuDraEnabled(); }
    bool readsPaths() const { return pcieTopologyAware || draEnabled() || vfVgpuDraEnabled() || resetCheck || aerPortHealth; }
    // DRA ResourceSlices of vGPUs on SR-IOV VFs (include/kxpu.h, kxpu_dra_slices_vf_vgpu): a vgpuDraDriver on a vfVgpu
    // class publishes its vGPUs (VfVgpuResourceSlices) in the pool nodeName.  With one set, the PCI gathers read
    // numa_node and the entry link as draEnabled does, and readVfVgpus keeps each VF's physfn basename; nothing else is
    // read.  With none set, every read, output and generation is as without the setting.
    bool vfVgpuDraEnabled() const;  // some passthrough class has a vgpuDraDriver
    // DRA ResourceSlices of vGPUs (ABI v10): a draDriver on a vGPU class publishes its groups (VgpuResourceSlices) in
    // the pool nodeName.  With one set, the mdev walk also reads, for every entry that got as far as its iommu_group
    // link, the parent's numa_node (as topologyAware does), the entry's link (readPciPath) and <uuid>/../device; a failed
    // read only leaves out its attribute.  The PCI walk and every device-plugin output stay as they are.
    bool vgpuDraEnabled() const;  // some vGPU class has a draDriver
    bool readsMdevNuma() const { return topologyAware || vgpuDraEnabled(); }
    // the mdev walk reads each grouped entry's link (vgpuPcieTopologyAware, vgpuDraEnabled or aerPortHealth); one read
    // serves all
    bool readsMdevPaths() const { return vgpuPcieTopologyAware || vgpuDraEnabled() || aerPortHealth; }
    // DRA device taints (ABI v11).  false (default): the slices never carry taints and every output and generation is as
    // above, even while a device is Unhealthy.  true: ResourceSlices, VfVgpuResourceSlices and VgpuResourceSlices pass taint times to the
    // slice call (64 devices per slice); a group that refreshDraHealth found unhealthy carries the taint
    // <draDriver>/unhealthy=vfio-device-missing:NoSchedule since the time it was found so, and PrepareDraDevices refuses
    // it.
    bool draTaints = false;
    // the clock of refreshDraHealth, unix seconds; a seam (time(nullptr) when empty)
    std::function<int64_t()> now;
    // PCIe AER health (include/kxpu.h, ABI v12).  false (default): no aer_dev_* file is opened and every output is as
    // above.  true: after every walk and on refreshAerHealth, <bdf>/aer_dev_fatal and aer_dev_nonfatal of every accepted
    // PCI function and of every accepted mdev's parent (entry "<uuid>/.." under mdevBasePath) are read through
    // readAerFile, and a group where some member's count is above aerFatalLimit / aerNonFatalLimit gets Device::aer and
    // is sent Unhealthy.  Allocate does not refuse it: the kubelet does not hand out Unhealthy devices.  With draTaints
    // too, such a group is published with the taint <draDriver>/pcie-aer=fatal (else =nonfatal):NoSchedule, and
    // PrepareDraDevices prepares it, since a claim that tolerates the taint asked for it.  A function that is
    // re-enumerated starts with zeroed counters, so its taint clears at the next rediscover.
    bool aerHealth = false;
    // the non-fatal limit is separate because Unsupported Request errors count as non-fatal and some hosts see them often
    uint64_t aerFatalLimit = 0, aerNonFatalLimit = 0;
    // <base>/<entry>/<name>, at most KXPU_AER_FILE_MAX + 1 bytes; false or an empty out: a failed read (unknown count)
    std::function<bool(const std::string &base, const std::string &entry, const std::string &name, std::string &out)> readAerFile;
    // AER errors of the PCIe ports above a device (include/kxpu.h, kxpu_aer_ports and kxpu_aer_ports_mdev).  A Surprise
    // Down is logged by the downstream port above the device that dropped off the link, a completion timeout of a CPU read
    // by the root port, an error on a root port - switch link by the root port or the switch upstream port: none of them
    // in the device's own files [assumed, not observed here].  InitiateDevicePlugin refuses it while aerHealth is off.
    // false (default): no new link or file is read and every output, generation and counter is as above.  true:
    //   - the PCI walk reads every entry's link (as pcieTopologyAware does) and the mdev walk every grouped mdev's link
    //     (as readsMdevPaths), one read serving every setting that wants it, and each walk makes one kxpu_aer_ports /
    //     kxpu_aer_ports_mdev call after the gather, at start-up and on each rediscover (GroupState::aerPorts);
    //   - computeAer folds, after a group's members and PF, the aer_dev_* files of the ports above each member
    //     (<basePath>/<port>/aer_dev_fatal|nonfatal through readAerFile, counted in aerReads), one read per distinct port
    //     per call, with the same limits; the reason reads "<port> (PCIe port above <bdf>) reported <n> fatal ...";
    //   - a root port's count flags every group below it: errors are not traced further down.  The metrics' AER counts
    //     stay the group's own functions' and PF's; Unhealthy, the pcie-aer taint and the reason sample follow as for any
    //     AER flag, and refreshAerHealth re-reads the ports without a walk.
    bool aerPortHealth = false;
    // Restart resume of CDI indices (include/kxpu.h, ABI v13).  false (default): nothing more is read or written and every
    // index is the walk order of the first walk.  true: InitiateDevicePlugin reads back the CDI specs a previous process
    // wrote (<cdiConfigPath><cdiFileStem>.yaml of every class, kxpu_cdi_parse / kxpu_cdi_parse_mdev) and the index state
    // file <cdiConfigPath>.kata-xpu-cdi-index, and reconciles the first walks against them (kxpu_reconcile), so that a
    // function at the same bdf (a vGPU: the same UUID) in the same IOMMU group, whose group belongs to the same class file,
    // keeps the index its spec names.  The spec does not hold the device id, so a function whose model changed at the
    // same bdf and group keeps its index too; the runtime resolves the name to the same /dev/vfio/<g> either way.  Every
    // other function gets an index above every index handed out before.  A walk whose specs cannot be trusted (a file
    // that does not parse, an index or key in two entries, an index of 2^64-1) resumes from nothing known: fresh indices
    // from the state file's value (walk order without one), with a log line.  Start-up then writes the specs like
    // rediscover does (atomically, only when their bytes changed), and both start-up and rediscover keep the state file
    // current before any spec is written.  It rests on the kubelet reusing a restarted container's checkpointed
    // Allocate response [assumed].
    bool resumeIndices = false;
    const ResumeReport &resumeReport() const { return resume_; }
    // devices validated either way (tests, metrics).  The counters are atomic: Allocate counts under the shared lock, and
    // MetricsText reads them under it too
    std::atomic<uint64_t> liveValidations{0}, snapshotValidations{0};
    std::atomic<uint64_t> aerReads{0};  // aer_dev_* files read (tests, metrics)
    std::atomic<uint64_t> cdevReads{0};  // vfio-dev/ directories listed (tests, metrics)
    // SR-IOV virtual functions (include/kxpu.h, additions to ABI v14).  false (default): nothing named physfn or
    // sriov_numvfs is opened and every output is as above.  true: after either gather, physfn (readlink, basename) and
    // sriov_numvfs of every candidate of a passthrough class are read, and kxpu_sriov decides per group.  A group with a VF
    // whose PF is bound to a class driver ("<vf> needs the VF token of <pf> (bound to <driver>)": vfio-pci would ask for
    // the PF's VF token) or with a PF that has VFs enabled ("<pf> has <k> VFs enabled") goes through the blocker path:
    // sent Unhealthy, refused by Allocate and PrepareDraDevices, left out of the CDI spec and the DRA pool.  Allocate's live
    // path re-reads physfn, the PF's driver and sriov_numvfs.  With pcieTopologyAware the forest is kxpu_pcie_tree_sriov's,
    // so GetPreferredAllocation packs a request's VFs by PF.
    bool sriovAware = false;
    std::atomic<uint64_t> sriovReads{0};  // functions whose physfn and sriov_numvfs were read (tests, metrics)
    // Resets between tenants (include/kxpu.h, kxpu_reset_check).  false (default): no reset_method or reset file is opened
    // and every output, generation and counter is as above.  true: after either gather, the PCI walk reads the entry link
    // of every entry (as readsPaths), the `driver` link of every entry whose driver is not known yet (and `iommu_group` of
    // one bound to a class driver), and reset_method of every candidate of a passthrough class, falling back to whether
    // `reset` exists (kernels before 5.15).  A group with a member that has neither a method in resetMethods nor a
    // secondary-bus reset VFIO can do (every function below its parent bridge bound to a class driver and in its own
    // group) goes through the blocker path, with a reason naming the function ("0000:41:00.0 has no reset method in
    // resetMethods (reset_method: pm)", "... has no function reset and 0000:41:00.1 on its bus is bound to
    // snd_hda_intel", "... has no function reset and sits on a root bus"): sent Unhealthy, refused by Allocate and
    // PrepareDraDevices, left out of the CDI spec and every DRA pool.  rediscover reads everything again; Allocate reads
    // nothing more, since reset_method changes only when an administrator writes to it.  vGPU (mdev) groups are out of
    // scope: their reset is the vendor driver's.
    bool resetCheck = false;
    // the reset methods the plugin accepts: names of reset_method (flr, af_flr, pm, bus, cxl_bus, device_specific, acpi),
    // each at most once; InitiateDevicePlugin refuses any other.  A kernel without reset_method only counts with all seven.
    std::vector<std::string> resetMethods{"flr", "af_flr", "pm", "bus", "cxl_bus", "device_specific", "acpi"};
    // <base>/<bdf>/<name> for name "reset_method" (out: at most KXPU_RESET_FILE_MAX + 1 bytes) or "reset" (only whether
    // it exists: the file is write-only).  false with errno ENOENT: no such file; false with any other errno: a failed
    // read.  A seam: tests replace it.  Every call counts in resetReads.
    std::function<bool(const std::string &base, const std::string &bdf, const std::string &name, std::string &out)> readResetFile;
    std::atomic<uint64_t> resetReads{0};  // reset_method and reset files opened (tests, metrics)
    // <base>/<bdf>/nvidia/<name>, at most KXPU_VGPU_FILE_MAX + 1 bytes; false: the read failed ("no such file" included).
    // A seam: tests replace it.  Every call counts in vfVgpuReads.
    std::function<bool(const std::string &base, const std::string &bdf, const std::string &name, std::string &out)> readVgpuFile;
    std::atomic<uint64_t> vfVgpuReads{0};  // nvidia/ files read (tests, metrics)
    // Health of vGPUs on SR-IOV VFs (include/kxpu.h, kxpu_vf_vgpu_drift).  Refused by InitiateDevicePlugin unless some class
    // has vfVgpu.  false (default): no file more is opened and every output, generation and counter is as above.  true:
    //   - refreshVfVgpuTypes re-reads the type of every served VF and withholds one whose type changed;
    //   - the PCI walk keeps each VF's physfn basename (as vfVgpuDraEnabled does), and with aerHealth the PF's aer_dev_*
    //     files count as one more member of each group whose first member is a VF of a vfVgpu class: errors that no one
    //     function owns (a surprise down, a fatal link error, a completion timeout of the GPU) are logged on the PF;
    //   - with draTaints, a drifted group in a vgpuDraDriver pool carries <vgpuDraDriver>/vgpu-type=changed:NoSchedule,
    //     a fourth entry of that pool's taint table, and PrepareDraDevices refuses it.
    bool vfVgpuHealth = false;
    // mdev vGPUs on SR-IOV virtual functions (include/kxpu.h, kxpu_mdev_pf).  Refused by InitiateDevicePlugin unless some
    // vGPU class is configured.  On vGPU releases before the vendor-specific VFIO framework, an SR-IOV GPU's mdevs are
    // created on its VFs, so the mdev walk's parent is a VF.  false (default): nothing more is opened and every output,
    // generation and counter is as above.  true:
    //   - the mdev walk reads <uuid>/../physfn (readLink) of every entry that got as far as its iommu_group link, and
    //     kxpu_mdev_pf joins it to the PCI walk's records; a group whose first mdev's parent is a VF keeps its PF's
    //     address (GroupState::pf);
    //   - with aerHealth the PF's aer_dev_* files count as one more member of that group, each PF read once per call:
    //     errors of the whole GPU are logged on the PF, and a VF may have no files of its own;
    //   - VgpuResourceSlices publishes through kxpu_dra_slices_mdev_pf: such a vGPU carries physfnAddress, the PF's
    //     device id as physfnDeviceID and the PF's model name as productName, so claims can group or spread vGPUs by
    //     physical GPU.  A vGPU whose parent is not a VF is published exactly as without the setting.
    bool vgpuSriovAware = false;
    std::atomic<uint64_t> mdevPhysfnReads{0};  // <uuid>/../physfn links read (tests, metrics)
    // Passthrough SR-IOV VFs held to their PF (include/kxpu.h, kxpu_dra_slices_pf).  Refused by InitiateDevicePlugin
    // unless sriovAware is on, whose pf_of it reads.  It applies to the groups of passthrough classes without vfVgpu (an
    // AMD MxGPU VF, an Intel Flex / Max VF, a NIC VF on vfio-pci); a vfVgpu class keeps vfVgpuHealth's path.  false
    // (default): nothing more is opened and every output, generation and counter is as above.  true:
    //   - a group whose first member is a VF of a PF in the walk keeps that PF's address (GroupState::pf) and, with a
    //     draDriver, its device id: the PF's own record's, else its `device` file read once per walk (a PF on its
    //     vendor driver is no class candidate, so the gather left the id unread);
    //   - with aerHealth the PF's aer_dev_* files count as one more member of that group, each PF read once per call:
    //     errors of the whole device (a surprise down, a fatal link error, a completion timeout) are logged on the PF,
    //     and a VF may have no files of its own.  The reason names the PF, draTaints taints the group pcie-aer, and the
    //     metrics count the PF's errors;
    //   - ResourceSlices publishes through kxpu_dra_slices_pf: such a device carries physfnAddress and physfnDeviceID, so
    //     a claim can ask for VFs of one physical device or of different ones.  A function that is not a VF is published
    //     exactly as without the setting, and a rediscovery that changes a published VF's PF moves draGeneration().
    // Allocate, CDI specs, GetPreferredAllocation and ListAndWatch topology do not change.
    bool sriovPfAware = false;
    // PCIe root ports and switches in DRA (include/kxpu.h, kxpu_pcie_ports and kxpu_dra_slices_pcie): a DNS subdomain
    // that qualifies two more attributes of every passthrough DRA pool.  InitiateDevicePlugin refuses a value that is not
    // a lowercase DNS subdomain of at most 63 bytes, one equal to or under kubernetes.io or k8s.io, and any value while
    // no passthrough class has a draDriver.  Empty (default): no new call runs and every output, generation and counter
    // is as above.  Set:
    //   - each PCI walk makes one kxpu_pcie_ports call over the classify CSR, on the paths every DRA walk reads (no new
    //     file or link is read), and each group keeps its root port and switch (GroupState::rootPort / pcieSwitch);
    //   - ResourceSlices publishes every passthrough class through kxpu_dra_slices_pcie: a device carries
    //     <draPcieDomain>/pcieRootPort and <draPcieDomain>/pcieSwitch where they exist, one name for every class, so a
    //     claim can keep a GPU and a NIC VF of two DRA drivers under one root port or one switch (matchAttribute).  The
    //     PF attributes follow sriovPfAware as above;
    //   - a rediscovery that moves a published group under another root port or switch moves draGeneration().
    // Allocate, PrepareDraDevices, CDI specs, ListAndWatch, GetPreferredAllocation, metrics and the vGPU pools do not
    // change.
    std::string draPcieDomain;
    // PCIe root ports and switches of vGPUs in DRA (include/kxpu.h, kxpu_pcie_ports_mdev, kxpu_dra_slices_mdev_pcie and
    // kxpu_dra_slices_vf_vgpu_pcie): the vGPU pools publish <draPcieDomain>/pcieRootPort and <draPcieDomain>/pcieSwitch
    // too, so a claim can keep a vGPU and a NIC VF of another DRA driver under one switch.  A switch of its own, not
    // implied by draPcieDomain: with it off the vGPU pools' bytes are as above whatever draPcieDomain says.
    // InitiateDevicePlugin refuses it while draPcieDomain is empty, and while no vGPU class publishes DRA (no vGPU class
    // has a draDriver and no class a vgpuDraDriver).  false (default): no new call runs and every output, generation and
    // counter is as above.  true:
    //   - each mdev walk (with a vGPU class that has a draDriver) makes one kxpu_pcie_ports_mdev call over the classify
    //     CSR, on the links the DRA walk already reads (no new file or link is read); each group keeps the keys of its
    //     parent GPU (GroupState::rootPort / pcieSwitch);
    //   - VgpuResourceSlices publishes through kxpu_dra_slices_mdev_pcie, the physfn fields filled only with
    //     vgpuSriovAware and the PF's product as above; VfVgpuResourceSlices publishes through
    //     kxpu_dra_slices_vf_vgpu_pcie with the keys the PCI walk keeps for each group (no new call);
    //   - a rediscovery that moves a published mdev vGPU under another root port or switch moves draVgpuGeneration();
    //     one that moves a VF-vGPU moves draGeneration(), as for any group of the PCI walk.
    // Allocate, PrepareDraDevices, CDI specs, ListAndWatch, GetPreferredAllocation and the metrics do not change.
    bool draVgpuPcie = false;
    // (type ID, type key) of every vGPU type a walk of this process named: the last name table of kxpu_vf_vgpu_types, so a
    // GPU that became full keeps its names across rediscover
    const std::map<uint32_t, std::string> &learnedVgpuTypes() const { return learnedVgpuTypes_; }
    bool vfVgpuEnabled() const;  // some passthrough class has vfVgpu
    bool cdevEnabled() const;  // some passthrough class has vfioCdev
    bool mdevCdevEnabled() const;  // some vGPU class has mdevCdev

    // ---- state (device_plugin.go:31,34)
    OrderedMap<std::vector<NvidiaGpuDevice>> iommuMap;  // group id -> devices
    OrderedMap<std::vector<std::string>> deviceMap;     // device id -> iommu groups
    // a deque: a rediscovery appends plugins without moving the others (HealthWatcher holds a reference)
    std::deque<GenericDevicePlugin> devicePlugins;
    std::string lastCdiFile;
    std::vector<GroupState<kxpu_dradev>> iommuState;  // the state of every iommuMap entry (same positions)
    std::vector<size_t> deviceClass;  // class of every deviceMap entry (same positions); all 0 with the default class list
    std::vector<bool> deviceNamed;    // deviceMap entry keyed by a configured resource name (same positions)
    // pcieTopologyAware only: the forest of the last PCI walk, shared by all passthrough plugins
    std::vector<uint32_t> pcieParent;
    std::vector<uint8_t> pcieDepth;
    std::vector<std::string> cdiFiles;  // files the last generateCDISpec wrote, one per class
    // the mdev walk: IOMMU group -> mdevs and type key -> groups, the state of every mdevMap entry and the vGPU class of
    // every typeMap entry (same positions)
    OrderedMap<std::vector<MdevDevice>> mdevMap;
    OrderedMap<std::vector<std::string>> typeMap;
    std::vector<GroupState<kxpu_dramdev>> mdevState;
    std::vector<size_t> typeClass;
    // vgpuPcieTopologyAware only: the forest of the last mdev walk, shared by all vGPU plugins
    std::vector<uint32_t> mdevPcieParent;
    std::vector<uint8_t> mdevPcieDepth;
    std::vector<std::string> mdevCdiFiles;  // files the last generateMdevCDISpec wrote, one per vGPU class

    explicit Plugin(kxpu_ctx *ctx);
    ~Plugin();

    // device_plugin.go:44-53 without the blocking gRPC part
    Error InitiateDevicePlugin();
    // device_plugin.go:126-180: walk + raw gather on the host, classify on the GPU (S1)
    Error createIommuDeviceMap();
    // device_plugin.go:208-259: parse-once table + batched lookup + sanitiser on the GPU (S2)
    std::string getDeviceName(const std::string &deviceID);
    // the same for a batch of ids: one kxpu_lookup + one kxpu_names (device_plugin.go:99 for every id of deviceMap);
    // vendors[i] is the vendor id of deviceIDs[i]
    std::vector<std::string> getDeviceNames(const std::vector<std::string> &deviceIDs, const std::vector<std::string> &vendors);
    // device_plugin.go:55-80 + cdi/spec.go:85-127: emit on the GPU, host writes the file (S3)
    Error generateCDISpec(const OrderedMap<std::vector<NvidiaGpuDevice>> &m, const std::string &format = "YAML");
    // the mdev walk (single-threaded, lexical order) + kxpu_classify_mdev; reads nothing when vgpuClasses is empty
    Error createMdevMap();
    // one CDI spec per vGPU class (kxpu_cdi_emit_mdev), <stem>.yaml|.json; nothing when vgpuClasses is empty
    Error generateMdevCDISpec(const std::string &format = "YAML");
    // device_plugin.go:83-112: per device id device lists + plugin objects (S4), then one plugin per (vGPU class, type
    // key); nothing is started
    Error createDevicePlugins();
    // generic_device_plugin.go:320-355 for one container request (S5).  groupViability: a group the last walk found not
    // viable fails the request before any read
    Error Allocate(const std::vector<std::string> &devicesIDs, ContainerAllocateResponse &resp);
    // generic_device_plugin.go:224: the bytes of ListAndWatchResponse{Devices: dpi.devs}
    Error ListAndWatchBytes(const GenericDevicePlugin &dp, std::vector<uint8_t> &out);
    // generic_device_plugin.go:253-258: GetPreferredAllocationAvailable = topologyAware || pcieTopologyAware ||
    // vgpuPcieTopologyAware
    DevicePluginOptions GetDevicePluginOptions() const;
    // generic_device_plugin.go:378-386 (the reference: nil, nil).  topologyAware: one kxpu_preferred_allocation call for
    // all container requests, device IDs mapped to positions in dp.devs; an ID not in dp.devs is an error naming it.
    Error GetPreferredAllocation(const GenericDevicePlugin &dp, const std::vector<ContainerPreferredAllocationRequest> &requests,
                                 std::vector<ContainerPreferredAllocationResponse> &responses);

    // Runtime rediscovery (include/kxpu.h, kxpu_reconcile).  Under an exclusive lock (Allocate, ListAndWatchBytes and
    // GetPreferredAllocation take it shared): read the uevent generations, walk and classify as at start-up, reconcile
    // each walk against its snapshot (a surviving function or mdev keeps its CDI index, every other one gets an index
    // never handed out before), rebuild the maps, rewrite each CDI spec whose bytes changed (atomically), update
    // devicePlugins in place (matched by vgpu, class and device key; health carried per group, new groups Healthy, new
    // plugins appended, a plugin whose devices all left keeps an empty list) and take a fresh snapshot generation.
    // A restart numbers by walk order again unless resumeIndices is on.
    Error rediscover(RediscoverReport &report, const std::string &format = "YAML");
    // The ResourceSlices of class xpuClass (kxpu_dra_slices): one pool named nodeName, one device per iommuMap group of
    // the class in walk order (bdf, vendor, device and PCIe root of the group's first member, the group's NUMA mask, the
    // plugin's resource-name suffix -- with resourceNames the group's model name, Device::model -- cut to 64 bytes as
    // productName).  With groupViability a group that has a blocker is
    // not published, also with draTaints: a taint can be tolerated, and on a cluster without the DRADeviceTaints feature
    // gate a tainted device looks healthy, so a group VFIO cannot open would be handed out.  Without draTaints health
    // from the HealthWatcher is not consulted; with it, a group refreshDraHealth found unhealthy is published tainted.
    // out: JSON Lines, one slice per line; sliceOff: the n_slices + 1 line bounds.
    Error ResourceSlices(size_t xpuClass, std::vector<uint8_t> &out, std::vector<uint64_t> &sliceOff);
    // the pool generation of every class's ResourceSlices: 1 after start-up, +1 for each rediscover that changed a
    // passthrough plugin or a group's viability, +1 for each refreshDraHealth that changed their taints; the VF-vGPU
    // pools (VfVgpuResourceSlices) share it, their VFs being functions of the PCI walk
    uint64_t draGeneration() const { return pci_.draGeneration; }
    // draTaints: the device-plugin health of every group published in a DRA pool becomes its taint.  The host calls it
    // after HealthWatcher::poll returned > 0.  Under the exclusive lock: a group that any plugin serving it has
    // Unhealthy is tainted since now() when it turns unhealthy, keeps that time while it stays so and loses it when it
    // turns healthy; draGeneration / draVgpuGeneration grow by one when the taints of their pools changed, and
    // passthroughMoved / vgpuMoved say which did.  Without draTaints nothing changes.
    Error refreshDraHealth(bool &passthroughMoved, bool &vgpuMoved);
    // aerHealth: re-read every AER file and fold the counts again (kxpu_aer_health), with no walk, under the exclusive
    // lock.  Sysfs attributes send no inotify or uevent, so the host calls this on a timer.  changedPlugins: the plugins
    // whose ListAndWatch bytes changed; with draTaints, passthroughMoved / vgpuMoved say which pools' AER taints changed
    // (their generation grew by one).  Without aerHealth nothing is read and nothing changes.
    Error refreshAerHealth(std::vector<size_t> &changedPlugins, bool &passthroughMoved, bool &vgpuMoved);
    // vfVgpuHealth: re-read nvidia/current_vgpu_type (readVgpuFile) of the VF each vfVgpu plugin device stands for (the
    // first member of its group; free VFs are not read) and compare it with the walk's type (kxpu_vf_vgpu_drift), under
    // the exclusive lock.  Writing the file sends no event, so the host calls this on a timer, like refreshAerHealth.  A
    // VF whose type is cleared, changed or unreadable gets Device::drift and is sent Unhealthy; one that reads back its
    // walk's type loses it.  changedPlugins: the plugins whose ListAndWatch bytes changed; passthroughMoved: the taints
    // of a VF-vGPU pool changed (draGeneration grew by one); typesMoved: some served VF carries another non-zero type, so
    // a rediscover would now move it to that type's resource.  The maps, indices and specs are never rebuilt here.
    // Without vfVgpuHealth nothing is read and nothing changes.
    Error refreshVfVgpuTypes(std::vector<size_t> &changedPlugins, bool &passthroughMoved, bool &typesMoved);
    // The Prometheus text (format 0.0.4, include/kxpu.h) of the current plugins and group state, under the shared lock:
    // one kxpu_metrics_devices call for every device of every plugin in devicePlugins order (whether ListAndWatch sends
    // it Healthy, each reason the host holds for it, its group's AER maxima), then the host's read and validation
    // counters.  It reads nothing from sysfs and changes no state: it reports what the last walk and refreshes found.  A
    // host that serves GET /metrics calls it per scrape.  A label string longer than KXPU_METRICS_STRING_MAX bytes is cut
    // there (metricsCut), so one long reason cannot make the whole scrape fail.
    Error MetricsText(std::vector<uint8_t> &out);
    // The ResourceSlices of the vGPUs of vfVgpu class xpuClass (kxpu_dra_slices_vf_vgpu): one pool named nodeName, one
    // device per iommuMap group of the class in walk order whose first member is a VF that carries a named vGPU type,
    // unless the group has a blocker (as ResourceSlices).  The device is described by that VF: its address, type key and
    // type ID, the PCIe root of its link, the group's NUMA mask, and its PF (the physfn basename): the PF's address, the
    // vendor and device ids of the PF's record in the same walk (a PF the walk did not read: the VF's vendor id and no
    // device id), and the PF's model name (getDeviceNames: the sanitised pci.ids name, else the raw device id; cut to 64
    // bytes) as productName.  Generation: draGeneration, since these VFs are functions of the PCI walk; taints as for
    // ResourceSlices.
    Error VfVgpuResourceSlices(size_t xpuClass, std::vector<uint8_t> &out, std::vector<uint64_t> &sliceOff);
    // The ResourceSlices of vGPU class vgpuClass (kxpu_dra_slices_mdev): one pool named nodeName, one device per mdevMap
    // group of the class in walk order, described by the group's first mdev: its type key, UUID, parent address, the
    // parent's vendor and device ids, the PCIe root of its link, the group's NUMA mask, and the parent's model name
    // (getDeviceNames: the sanitised pci.ids name, else the raw device id; cut to 64 bytes) as productName.
    Error VgpuResourceSlices(size_t vgpuClass, std::vector<uint8_t> &out, std::vector<uint64_t> &sliceOff);
    // the pool generation of every vGPU class's ResourceSlices: 1 after start-up, +1 for each rediscover that changed a
    // vGPU plugin, +1 for each refreshDraHealth that changed their taints
    uint64_t draVgpuGeneration() const { return mdev_.draGeneration; }
    // The data half of NodePrepareResources: cdiIds[i] = the CDI names Allocate({g}) returns for deviceNames[i] =
    // "vfio<g>", a device of the pool `pool` of the class (passthrough or vGPU) whose draDriver is `driver`, or of the vfVgpu
    // class whose vgpuDraDriver it is (same live or snapshot re-validation, same viability refusal; a vGPU group is always
    // re-read live, and Allocate refuses a VF whose vGPU type changed since the walk).  An unknown driver, pool or
    // device is an error that names it.
    Error PrepareDraDevices(const std::string &driver, const std::string &pool, const std::vector<std::string> &deviceNames,
                            std::vector<std::vector<std::string>> &cdiIds);

    // has a pci (or, with vGPU classes, an mdev) uevent generation moved since the last walk?  true when it cannot tell
    bool discoveryStale();
    // the snapshot of the last walks (kxpu_snaprec per accepted function / mdev in walk order) and their next index
    const std::vector<kxpu_snaprec> &pciSnapshot() const { return pci_.snap; }
    const std::vector<kxpu_snaprec> &mdevSnapshot() const { return mdev_.snap; }
    uint64_t pciNextIndex() const { return pci_.next; }
    uint64_t mdevNextIndex() const { return mdev_.next; }

    // raw gather only (no GPU): exposed for CPU tests of the walk.  paths (pcieTopologyAware only, else left empty):
    // one kxpu_pcipath per record, same index
    // cdevs (cdevEnabled only, else left empty): per record N of its VFIO cdev, -1 = none or not read
    // srs (sriovAware only, else left empty): per record its physfn and sriov_numvfs reads, zero-filled for a record that
    // is no candidate of a passthrough class
    Error gatherRecords(std::vector<kxpu_devrec> &recs, std::vector<kxpu_pcipath> *paths = nullptr,
                        std::vector<int64_t> *cdevs = nullptr, std::vector<kxpu_sriovrec> *srs = nullptr);
    // the same records, read with openat / readlinkat relative to basePath by several threads
    // (SURVEY 8(f) row 2); falls back to gatherRecords when a seam was replaced.  threads = 0: automatic
    Error gatherRecordsFast(std::vector<kxpu_devrec> &recs, unsigned threads = 0, std::vector<kxpu_pcipath> *paths = nullptr,
                            std::vector<int64_t> *cdevs = nullptr, std::vector<kxpu_sriovrec> *srs = nullptr);
    // physfn (readlink, basename) and the first 8 bytes of sriov_numvfs of <basePath>/<bdf>; a missing link or file is
    // no error, any other failure sets KXPU_SR_PHYSFN_ERR / KXPU_SR_NUMVFS_ERR.  Counts in sriovReads.
    kxpu_sriovrec readSriov(const std::string &bdf);
    // the cdev of <base>/<entry> (a function's bdf under basePath, an mdev's uuid under mdevBasePath): N when vfio-dev/
    // holds exactly one entry besides . and .., and it is "vfio" followed by a canonical decimal below 2^32; -1 for
    // anything else (never an error)
    int64_t readVfioCdev(const std::string &base, const std::string &entry);
    // raw gather of mdevBasePath under vgpuClasses (no GPU): one record per entry, lexical order.  w (vgpuDraEnabled
    // only, else left empty): the walk's parentDevice and pcieRoot, one per record; (readsMdevPaths only, else left
    // empty) its paths; (mdevCdevEnabled only, else left empty) its cdevs
    Error gatherMdevRecords(std::vector<kxpu_mdevrec> &recs, MdevWalk *w = nullptr);
    // resetCheck: the reads kxpu_reset_check needs after a gather (no GPU): the driver (and iommu_group) of every entry
    // that lacks it into recs, and one kxpu_resetrec per record into rrs, zero-filled for a record that is no candidate of
    // a passthrough class.  Off: rrs is left empty and nothing is read.
    void readResets(std::vector<kxpu_devrec> &recs, std::vector<kxpu_resetrec> &rrs);
    // the vGPU class list against the passthrough one (distinct CDI kinds and file stems, no vfioCdev on a vGPU class, no
    // mdevCdev on a passthrough class); createMdevMap runs it
    Error checkVgpuClasses() const;
    // the gather with the vfVgpu reads (no GPU): w.vts and w.creatable, one per record
    Error gatherVfVgpu(PciWalk &w);

  private:
    kxpu_ctx *ctx_;
    kxpu_table *table_ = nullptr;
    Error ensureTable();
    Error gatherRecordsFastWalk(std::vector<kxpu_devrec> &recs, unsigned threads, std::vector<kxpu_pcipath> *paths);
    void readCdevs(const std::vector<kxpu_devrec> &recs, std::vector<int64_t> *cdevs);
    void readSriovs(const std::vector<kxpu_devrec> &recs, std::vector<kxpu_sriovrec> *srs);
    std::map<uint32_t, std::string> learnedVgpuTypes_;
    std::string pfDeviceOf(const kxpu_devrec &pf, std::map<std::string, std::string> &read) const;
    std::vector<kxpu_devrec> pciRecs_;  // vgpuSriovAware only: the last PCI walk's records, which kxpu_mdev_pf joins against
    // vfVgpu: the nvidia/ reads of every VF of such a class into w, then the type join (kxpu_vf_vgpu_types)
    void readVfVgpus(PciWalk &w);
    Error joinVgpuTypes(PciWalk &w);
    // the classes whose functions are passed through whole: xpuClasses, a vfVgpu class's driver counting as none
    bool passthroughDriver(const std::string &driver) const;
    Error checkVfVgpuClasses() const;
    // resourceNames: each key and value well formed, no name on two classes, at most KXPU_MAX_NAMES entries, none on a
    // vfVgpu or vGPU class; InitiateDevicePlugin runs it
    Error checkResourceNames() const;
    // the name table of kxpu_classify_named over xpuClasses (one slot per distinct (class, name), in class and key
    // order) and the name of each slot
    void nameTable(std::vector<kxpu_name_entry> &entries, std::vector<std::string> &slotNames) const;
    // resetMethods against the seven names; InitiateDevicePlugin runs it
    Error checkResetMethods() const;
    uint32_t resetAllow() const;  // resetMethods as KXPU_RM_* bits
    std::string resetReasonOf(const PciWalk &w, uint32_t i) const;  // the reason of kxpu_reset_check's blocker i
    // Allocate's live SR-IOV check of one function: the reason kxpu_sriov's rule now gives, or ""
    std::string sriovLive(const std::string &bdf);
    // one CDI spec per class: the devices of m whose entry has that class (entryClass, same positions as m)
    template <typename Dev, typename Rec>
    Error generateClassSpecs(const std::vector<XpuClass> &classes, const OrderedMap<std::vector<Dev>> &m,
                             const std::vector<size_t> &entryClass, int32_t fmt, const char *what,
                             int32_t (*emit)(kxpu_ctx *, int32_t, const char *, const Rec *, size_t, uint8_t *, size_t, size_t *),
                             std::vector<std::string> &files);
    // first use: kxpu_pciids_join on pinned buffers = file -> table -> row handles of `keys` in one call
    Error loadAndJoin(const std::vector<uint32_t> &keys, std::vector<int32_t> &rows);
    // One walk's bookkeeping between its walks: pci_ for the PCI functions, mdev_ for the mdevs
    struct WalkBook {
        std::vector<kxpu_snaprec> snap;  // the last walk's snapshot: one kxpu_snaprec per accepted entry, walk order
        uint64_t next = 0;               // the next CDI index
        bool haveGen = false;            // the uevent generation read before the last walk, when it could be read
        uint64_t gen = 0;
        uint64_t draGeneration = 1;      // the generation of the walk's DRA pools
        // whether source still returns the generation read before the last walk; false when it cannot tell
        bool current(const std::function<bool(uint64_t &generation)> &source) const {
            uint64_t g = 0;
            return haveGen && source && source(g) && g == gen;
        }
    };
    WalkBook pci_, mdev_;
    // the walk and classify of one kind of walk
    Error classify(PciWalk &w);
    Error classify(MdevWalk &w);
    // iommuMap / deviceMap (mdevMap / typeMap) of a walk; index == nullptr: busIndex, else index[busIndex]
    void buildMaps(const PciWalk &w, const std::vector<uint64_t> *index);
    void buildMaps(const MdevWalk &w, const std::vector<uint64_t> *index);
    std::vector<kxpu_snaprec> snapshotOf(const PciWalk &w, const std::vector<uint64_t> *index) const;
    std::vector<kxpu_snaprec> snapshotOf(const MdevWalk &w, const std::vector<uint64_t> *index) const;
    // the first walk of createIommuDeviceMap / createMdevMap: classify, the maps with walk-order indices, and the record
    template <typename Walk>
    Error firstWalk(Walk &w, WalkBook &book);
    // rediscover: classify, reconcile against the record's snapshot (a surviving entry keeps its index, every other one
    // gets an index never handed out before), then the maps with the reconciled indices
    template <typename Walk>
    Error rewalk(Walk &w, WalkBook &book, kxpu_reconcile_counts &counts);
    Error buildPlugins(std::vector<GenericDevicePlugin> &out);
    // resumeIndices: the previous specs' entries of one walk and its next index, from the state file and the specs
    template <typename Rec>
    void previousEntries(const std::vector<XpuClass> &classes,
                         int32_t (*parse)(kxpu_ctx *, int32_t, const char *, const uint8_t *, size_t, Rec *, size_t, size_t *),
                         uint64_t stateNext, ResumeWalk &rw, std::vector<kxpu_snaprec> &prev, uint64_t &next);
    // resumeIndices: reconcile the first walk's entries `cur` (klass = the class of the entry's group, tag 0 but for the
    // vGPU VFs of a class whose spec was read typed) against the previous specs; index gets one index per cur entry,
    // nextOut the walk's next index
    Error resumeWalk(std::vector<kxpu_snaprec> prev, uint64_t next, uint64_t stateNext, const std::vector<kxpu_snaprec> &cur,
                     ResumeWalk &rw, std::vector<uint64_t> &index, uint64_t &nextOut);
    // resumeIndices: the first walk against the previous specs' entries prev (next: their next index, stateNext the state
    // file's value); rebuilds the walk's maps and record with the resumed indices
    template <typename Walk>
    Error resume(const Walk &w, WalkBook &book, ResumeWalk &rw, uint64_t stateNext, std::vector<kxpu_snaprec> prev,
                 uint64_t next);
    void readIndexState();  // into resume_
    Error writeIndexState(std::vector<std::string> *written);
    ResumeReport resume_;
    bool atomicSpecs_ = false;  // rediscover: specs are written only when changed, through .tmp + fsync + rename
    std::vector<std::string> specsWritten_;
    Error writeSpec(const std::string &path, const std::vector<uint8_t> &doc, size_t len, bool &written);
    mutable std::shared_mutex mu_;
    BindWatcher bindWatcher_;
    bool haveSnapshotGen_ = false;
    uint64_t snapshotGen_ = 0;
    std::map<std::string, int64_t> draTaintSince_;  // draTaints: IOMMU group id -> when its taint was added
    // draTaints && aerHealth: IOMMU group id -> (KXPU_AER_FATAL or KXPU_AER_NONFATAL, when that value was first seen)
    std::map<std::string, std::pair<uint8_t, int64_t>> aerTaint_;
    // draTaints && vfVgpuHealth: IOMMU group id -> when refreshVfVgpuTypes first saw its VF drift (the vgpu-type taint)
    std::map<std::string, int64_t> driftTaint_;
    Error computeAer();  // the reads and the kxpu_aer_health call for the current maps, into their states' aer / aerBits
    // aerTaint_ from the last computeAer for the groups the DRA pools publish; which pools' taints changed
    void updateAerTaints(bool &passthroughMoved, bool &vgpuMoved);
    // per group its time in draTaintSince_, then with aerHealth (or typeTaint) its pcie-aer=fatal and =nonfatal times,
    // then with typeTaint its time in driftTaint_; -1: no such taint
    std::vector<int64_t> draSinceTable(const std::vector<std::string> &groups, bool typeTaint) const;
    // one pool's slices of devs, the records of groups, through fn (kxpu_dra_slices_taints or _mdev_taints) with the
    // table <driver>/unhealthy=vfio-device-missing, then with aerHealth <driver>/pcie-aer=fatal and =nonfatal, then with
    // typeTaint (a VF-vGPU pool under vfVgpuHealth) all three and <driver>/vgpu-type=changed, all NoSchedule; without
    // draTaints taint_since is NULL (the untainted bytes)
    // fn: a slice call of the taint-list form (kxpu_dra_slices_taints' signature for Rec), or one wrapping such a call
    template <typename Rec, typename Fn>
    Error draSlices(Fn fn, const char *what, const std::string &driver, uint64_t generation, const std::vector<Rec> &devs,
                    const std::vector<std::string> &groups, std::vector<uint8_t> &out, std::vector<uint64_t> &sliceOff,
                    bool typeTaint = false) const;
    Error checkDraClasses() const;
    Error checkDraPcieDomain() const;
    Error checkDraVgpuPcie() const;
    void buildMdevDra(const MdevWalk &w);
    void buildVfVgpuDra(const PciWalk &w);
};

}  // namespace device_plugin
