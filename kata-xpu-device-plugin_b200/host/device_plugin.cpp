// device_plugin.cpp -- see device_plugin.hpp.  Reference: pkg/device_plugin/device_plugin.go,
// pkg/device_plugin/generic_device_plugin.go, cdi/spec.go (citations per function).
#include "device_plugin.hpp"

#include <dirent.h>
#include <poll.h>
#include <linux/netlink.h>
#include <sys/inotify.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <unistd.h>

#include <fcntl.h>

#include <climits>
#include <mutex>

#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <set>
#include <thread>
#include <type_traits>

namespace device_plugin {

static const char *kDevicePluginPath = "/var/lib/kubelet/device-plugins/";  // pluginapi.DevicePluginPath
static const char *kHealthy = "Healthy";                                     // pluginapi.Healthy
static const char *kUnhealthy = "Unhealthy";                                 // pluginapi.Unhealthy
static const char *kK8SCDIVendorClass = "KUBERNETES_CDI_VENDOR_CLASS";       // generic_device_plugin.go:29
static const char *kCdiVendorClass = "nvidia.com/gpu";                       // generic_device_plugin.go:30

XpuClass defaultXpuClass() { return XpuClass{"10de", "vfio-pci", "nvidia.com", kCdiVendorClass, "cdi-vfio-xxxx"}; }

// What ListAndWatch sends a device: Healthy only while the watcher has its node, the last walk found its group viable,
// its link reports no errors over the limits and (a VF) its vGPU type is the walk's.  MetricsText reports the same bit.
static bool sentHealthy(const Device &d) { return d.Health == kHealthy && d.blocker.empty() && d.aer.empty() && d.drift.empty(); }

static Error fail(const std::string &m) { Error e; e.failed = true; e.message = m; return e; }
static Error kxfail(kxpu_ctx *ctx, const char *what, int32_t rc) {
    return fail(std::string(what) + ": " + kxpu_strerror(rc) + " (" + kxpu_last_error(ctx) + ")");
}

// readIDFromFileFunc, device_plugin.go:183-191 -- the os.ReadFile half.  Returns the RAW file
// bytes: the data[2:] / Trim("\n") half of :189 runs on the GPU (kxpu_classify).
static bool readIDFromFileFunc(const std::string &base, const std::string &addr, const std::string &prop, std::string &out) {
    std::string path = base + "/" + addr + "/" + prop;  // filepath.Join
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) {
        fprintf(stderr, "Could not read %s for device %s: %s\n", prop.c_str(), addr.c_str(), strerror(errno));
        return false;
    }
    char buf[256];
    size_t n = fread(buf, 1, sizeof buf, f);
    bool err = ferror(f) != 0;
    fclose(f);
    if (err) return false;
    out.assign(buf, n);
    return true;
}

// readLinkFunc, device_plugin.go:194-202: os.Readlink + last path element.
static bool readLinkFunc(const std::string &base, const std::string &addr, const std::string &link, std::string &out) {
    std::string path = base + "/" + addr + "/" + link;
    char buf[4096];
    ssize_t n = readlink(path.c_str(), buf, sizeof buf - 1);
    if (n < 0) {
        fprintf(stderr, "Could not read link %s for device %s: %s\n", link.c_str(), addr.c_str(), strerror(errno));
        return false;
    }
    std::string target(buf, (size_t)n);
    size_t slash = target.find_last_of('/');  // filepath.Split
    out = slash == std::string::npos ? target : target.substr(slash + 1);
    return true;
}

// <base>/<entry>/numa_node, raw bytes.  Quiet: a missing file only means "node unknown".
static bool readNumaNodeFunc(const std::string &base, const std::string &entry, std::string &out) {
    const std::string path = base + "/" + entry + "/numa_node";
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) return false;
    char buf[64];
    size_t n = fread(buf, 1, sizeof buf, f);
    bool err = ferror(f) != 0;
    fclose(f);
    if (err) return false;
    out.assign(buf, n);
    return true;
}

// <base>/<entry>/<name>, at most KXPU_AER_FILE_MAX + 1 bytes (one more than a count is read from, so a longer file
// stays longer).  Quiet: a missing file only means "count unknown" (no AER capability, or a kernel before 4.19).
static bool readAerFileFunc(const std::string &base, const std::string &entry, const std::string &name, std::string &out) {
    const std::string path = base + "/" + entry + "/" + name;
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) return false;
    char buf[KXPU_AER_FILE_MAX + 1];
    size_t n = fread(buf, 1, sizeof buf, f);
    bool err = ferror(f) != 0;
    fclose(f);
    if (err) return false;
    out.assign(buf, n);
    return true;
}

static bool readVgpuFileFunc(const std::string &base, const std::string &bdf, const std::string &name, std::string &out) {
    FILE *f = fopen((base + "/" + bdf + "/nvidia/" + name).c_str(), "rb");
    if (!f) return false;
    std::vector<char> buf(KXPU_VGPU_FILE_MAX + 1);
    const size_t n = fread(buf.data(), 1, buf.size(), f);
    const bool err = ferror(f) != 0;
    fclose(f);
    if (err) return false;
    out.assign(buf.data(), n);
    return true;
}

// reset_method: its first KXPU_RESET_FILE_MAX + 1 bytes; reset: whether it exists (the file is write-only)
static bool readResetFileFunc(const std::string &base, const std::string &bdf, const std::string &name, std::string &out) {
    const std::string path = base + "/" + bdf + "/" + name;
    out.clear();
    if (name == "reset") {
        struct stat sb;
        return stat(path.c_str(), &sb) == 0;
    }
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) return false;
    char buf[KXPU_RESET_FILE_MAX + 1];
    const size_t n = fread(buf, 1, sizeof buf, f);
    const bool err = ferror(f) != 0;
    fclose(f);
    if (err) {
        errno = EIO;
        return false;
    }
    out.assign(buf, n);
    return true;
}

// the numa_node rule of include/kxpu.h: one trailing '\n' stripped, then a canonical decimal 0..63
static bool parseNumaNode(const std::string &raw, uint8_t &node) {
    std::string s = raw;
    if (!s.empty() && s.back() == '\n') s.pop_back();
    if (s.empty() || s.size() > 2 || (s.size() > 1 && s[0] == '0')) return false;
    unsigned v = 0;
    for (char c : s) {
        if (c < '0' || c > '9') return false;
        v = v * 10 + (unsigned)(c - '0');
    }
    if (v >= KXPU_MAX_NUMA_NODES) return false;
    node = (uint8_t)v;
    return true;
}
// readlink(<base>/<entry>): the whole target.  Quiet: a failed read only means "path unknown".
static bool readPciPathFunc(const std::string &base, const std::string &entry, std::string &out) {
    char buf[4096];
    ssize_t k = readlink((base + "/" + entry).c_str(), buf, sizeof buf);
    if (k < 0 || k == (ssize_t)sizeof buf) return false;
    out.assign(buf, (size_t)k);
    return true;
}

// the host rule of kxpu_pcipath: the target from its first component that begins with "pci"; none, or more than 120
// bytes from there, leaves the path unknown (len 0)
static void pciPathRecord(const std::string &target, kxpu_pcipath &p) {
    memset(&p, 0, sizeof p);
    for (size_t at = 0; at < target.size();) {
        if (target.compare(at, 3, "pci") == 0) {
            const size_t len = target.size() - at;
            if (len <= sizeof p.path) {
                memcpy(p.path, target.data() + at, len);
                p.len = (uint8_t)len;
            }
            return;
        }
        const size_t slash = target.find('/', at);
        if (slash == std::string::npos) return;
        at = slash + 1;
    }
}

template <typename ReadNuma>
static void numaRecord(ReadNuma readNuma, uint8_t &flags, uint8_t &node) {
    std::string s;
    uint8_t k = 0;
    if (readNuma(s) && parseNumaNode(s, k)) {
        node = k;
        flags |= KXPU_REC_NUMA;
    }
}

Plugin::Plugin(kxpu_ctx *ctx) : ctx_(ctx) {
    readNumaNode = readNumaNodeFunc;
    readAerFile = readAerFileFunc;
    readVgpuFile = readVgpuFileFunc;
    readResetFile = readResetFileFunc;
    readPciPath = readPciPathFunc;
    readLink = readLinkFunc;
    readIDFromFile = readIDFromFileFunc;
    returnIommuMap = [this]() -> const OrderedMap<std::vector<NvidiaGpuDevice>> & { return iommuMap; };
    returnMdevMap = [this]() -> const OrderedMap<std::vector<MdevDevice>> & { return mdevMap; };
    bindGeneration = [this](uint64_t &generation) {
        if (!bindWatcher_.healthy() && bindWatcher_.start()) return false;
        generation = bindWatcher_.generation();
        return bindWatcher_.healthy();
    };
    mdevGeneration = [this](uint64_t &generation) {
        if (!bindWatcher_.healthy() && bindWatcher_.start()) return false;
        generation = bindWatcher_.mdevGeneration();
        return bindWatcher_.healthy();
    };
}

// ---------------------------------------------------------------------------- bind / unbind uevents
BindWatcher::~BindWatcher() {
    if (fd_ >= 0) close(fd_);
}

Error BindWatcher::start() {
    if (fd_ >= 0) close(fd_);
    lost_ = false;
    fd_ = socket(AF_NETLINK, SOCK_DGRAM | SOCK_CLOEXEC | SOCK_NONBLOCK, NETLINK_KOBJECT_UEVENT);
    if (fd_ < 0) return fail(std::string("uevent socket: ") + strerror(errno));
    struct sockaddr_nl sa;
    memset(&sa, 0, sizeof sa);
    sa.nl_family = AF_NETLINK;
    sa.nl_groups = 1;  // kernel uevent multicast group
    if (bind(fd_, (struct sockaddr *)&sa, sizeof sa) != 0) {
        Error e = fail(std::string("uevent bind: ") + strerror(errno));
        close(fd_);
        fd_ = -1;
        return e;
    }
    return Error();
}

// "ACTION@DEVPATH\0KEY=VALUE\0..." -- a pci function changing its driver or coming / going
void BindWatcher::feed(const char *msg, size_t len) {
    const char *end = msg + len;
    std::string action, subsystem;
    for (const char *p = msg; p < end; p += strlen(p) + 1) {
        if (strncmp(p, "ACTION=", 7) == 0) action = p + 7;
        else if (strncmp(p, "SUBSYSTEM=", 10) == 0) subsystem = p + 10;
        if (memchr(p, 0, (size_t)(end - p)) == nullptr) break;  // unterminated tail
    }
    const bool moved = action == "bind" || action == "unbind" || action == "add" || action == "remove";
    if (subsystem == "pci" && moved) gen_++;
    else if (subsystem == "mdev" && moved) mdevGen_++;
}

uint64_t BindWatcher::generation() {
    if (fd_ < 0) return gen_;
    char buf[8192];
    for (;;) {
        ssize_t k = recv(fd_, buf, sizeof buf - 1, 0);
        if (k > 0) {
            buf[k] = 0;
            feed(buf, (size_t)k);
            continue;
        }
        if (k < 0 && errno == EINTR) continue;
        if (k < 0 && errno == ENOBUFS) { lost_ = true; gen_ += 1ull << 32; mdevGen_ += 1ull << 32; }  // messages were dropped
        break;
    }
    return gen_;
}

uint64_t BindWatcher::mdevGeneration() {
    generation();  // drains the socket: both counters are fed from the same messages
    return mdevGen_;
}

Plugin::~Plugin() {
    if (table_) kxpu_table_free(ctx_, table_);
}

// the Trim half of readIDFromFileFunc (:189): data[2:] with '\n' trimmed at both ends
static std::string trimID(const std::string &raw) {
    if (raw.size() < 2) return std::string();
    size_t a = 2, b = raw.size();
    while (a < b && raw[a] == '\n') a++;
    while (b > a && raw[b - 1] == '\n') b--;
    return raw.substr(a, b - a);
}

// an id file as the record carries it: the raw bytes when they fit the 8-byte field, else the
// canonical spelling "0x" + id + "\n" of the same id (identical after the reference's data[2:] /
// Trim); false when even that does not fit (the id itself is longer than 5 characters)
static bool packID(const std::string &raw, uint8_t txt[8], uint8_t &len) {
    if (raw.size() <= 8) {
        memcpy(txt, raw.data(), raw.size());
        len = (uint8_t)raw.size();
        return true;
    }
    const std::string id = trimID(raw);
    if (id.size() > 5 || id.find('\n') != std::string::npos) return false;
    const std::string canon = "0x" + id + "\n";
    memcpy(txt, canon.data(), canon.size());
    len = (uint8_t)canon.size();
    return true;
}

// The body of the walk callback for one non-directory entry (device_plugin.go:141-175, the reads
// only, in the reference's order and as lazily as the reference: nothing is read behind a vendor
// that no class has -- 10de by default -- or a driver that is not that vendor's class driver --
// vfio-pci by default): raw bytes of `vendor` / `device`, basenames
// of the `driver` / `iommu_group` links.  An entry the record cannot carry (address longer than 15
// bytes, group that is not a canonical decimal below 2^32-1, id longer than the field) is logged and
// skipped like a read error -- and only if the reference would have accepted it; it never stops the walk.
// readNuma == nullptr: numa_node is not read (Plugin::topologyAware false).  It is read last, only for a record that
// got as far as its device read, and changes nothing but numa_node / KXPU_REC_NUMA.
// allowed == nullptr: Plugin::groupViability false.  Otherwise an entry the class test rejected is a blocker when its
// driver (the `driver` link, read here if the class test did not read it) is bound and not in *allowed: the record then
// carries its `iommu_group` and driver and KXPU_REC_BLOCKS.  An unbound entry (failed read) is not a blocker; a group
// link outside the record's domain is logged and leaves the record as it is.
static bool parseGroup(const std::string &s, uint32_t &v);
template <typename ReadID, typename ReadLnk, typename ReadNuma>
static Error leafRecord(const std::string &name, const std::vector<XpuClass> &classes, ReadID readID, ReadLnk readLnk,
                        const ReadNuma *readNuma, const std::vector<std::string> *allowed, kxpu_devrec &r) {
    memset(&r, 0, sizeof r);
    strncpy(r.bdf, name.c_str(), sizeof r.bdf - 1);
    std::string s;
    // drv: the driver's basename when the class test read it already
    auto viability = [&](const std::string *drv) {
        if (!allowed) return Error();
        std::string d, g;
        if (drv) d = *drv;
        else if (!readLnk("driver", d)) return Error();
        if (std::find(allowed->begin(), allowed->end(), d) != allowed->end()) return Error();
        uint32_t v = 0;
        if (!readLnk("iommu_group", g) || !parseGroup(g, v)) {
            fprintf(stderr, "%s is bound to %s but its iommu_group is not a canonical decimal below 2^32-1: viability unknown\n",
                    name.c_str(), d.c_str());
            return Error();
        }
        r.iommu_group = v;
        memset(r.driver, 0, sizeof r.driver);
        memcpy(r.driver, d.data(), std::min<size_t>(d.size(), sizeof r.driver - 1));
        r.flags |= KXPU_REC_BLOCKS;
        return Error();
    };
    if (!readID("vendor", s)) {
        r.flags |= KXPU_REC_VENDOR_ERR;  // "Could not get vendor ID for device" -> skipped (:143-146)
        return viability(nullptr);
    }
    const std::string vendor = trimID(s);
    bool known = false;  // :149 -- the vendor of some class
    for (const XpuClass &c : classes) known = known || vendor == c.vendor;
    if (!packID(s, r.vendor_txt, r.vendor_len)) {  // an id of six or more characters is not 10de
        memcpy(r.vendor_txt, s.data(), 8);
        r.vendor_len = 8;
        r.flags |= KXPU_REC_VENDOR_ERR;
    }
    if (!known) return viability(nullptr);
    if (!readLnk("driver", s)) {
        r.flags |= KXPU_REC_DRIVER_ERR;  // :152-155
        return Error();
    }
    memcpy(r.driver, s.data(), std::min<size_t>(s.size(), sizeof r.driver - 1));
    bool bound = false;  // :156 -- the driver of that vendor's class
    for (const XpuClass &c : classes) bound = bound || (vendor == c.vendor && s == c.driver);
    if (!bound) return viability(&s);
    if (name.size() > sizeof r.bdf - 1) {
        fprintf(stderr, "PCI address longer than 15 bytes, device skipped: %s\n", name.c_str());
        r.flags |= KXPU_REC_IOMMU_ERR;
        return Error();
    }
    if (readLnk("iommu_group", s)) {  // :157
        bool dec = !s.empty() && s.size() <= 10;
        unsigned long long v = 0;
        for (char c : s) { if (c < '0' || c > '9') dec = false; else v = v * 10 + (unsigned)(c - '0'); }
        if (!dec || v >= 0xFFFFFFFFull || (s.size() > 1 && s[0] == '0')) {
            fprintf(stderr, "iommu_group of %s is not a canonical decimal number below 2^32-1, device skipped: %s\n", name.c_str(), s.c_str());
            r.flags |= KXPU_REC_IOMMU_ERR;
            return Error();
        }
        r.iommu_group = (uint32_t)v;
    } else {
        r.flags |= KXPU_REC_IOMMU_ERR;  // :158-161
        return Error();
    }
    // :164 reads `device` only for the first member of a group; which record that is is decided on
    // the GPU, so the file is read for every accepted candidate (a failure only matters for a first member)
    if (readID("device", s)) {
        if (!packID(s, r.device_txt, r.device_len)) {
            fprintf(stderr, "device id of %s is longer than the record field, device skipped\n", name.c_str());
            r.flags |= KXPU_REC_DEVICE_ERR;
        }
    } else {
        r.flags |= KXPU_REC_DEVICE_ERR;  // :165-168
    }
    if (readNuma) numaRecord(*readNuma, r.flags, r.numa_node);
    return Error();
}

// groupViability: the drivers that leave a group viable (viabilityDrivers and every class driver); nullptr when off
static const std::vector<std::string> *allowedDrivers(const Plugin &p, std::vector<std::string> &buf) {
    if (!p.groupViability) return nullptr;
    buf = p.viabilityDrivers;
    for (const XpuClass &c : p.xpuClasses) buf.push_back(c.driver);
    return &buf;
}

// filepath.Walk(basePath, ...) (device_plugin.go:132): lexical order, os.Lstat (symlinks are not
// followed, so a real sysfs entry is "not a directory"), directories are descended into and
// reported as "Not a device" (:137-140).
static Error walkDir(Plugin &p, const std::string &path, const std::string &name, std::vector<kxpu_devrec> &recs,
                     std::vector<kxpu_pcipath> *paths) {
    struct stat sb;
    if (lstat(path.c_str(), &sb) != 0) return fail("Error accessing file path \"" + path + "\": " + strerror(errno));  // :133-136
    if (S_ISDIR(sb.st_mode)) {
        DIR *d = opendir(path.c_str());
        if (!d) return fail("Error accessing file path \"" + path + "\": " + strerror(errno));
        std::vector<std::string> names;
        while (struct dirent *de = readdir(d)) {
            if (strcmp(de->d_name, ".") == 0 || strcmp(de->d_name, "..") == 0) continue;
            names.push_back(de->d_name);
        }
        closedir(d);
        std::sort(names.begin(), names.end());
        for (const std::string &n : names) {
            Error e = walkDir(p, path + "/" + n, n, recs, paths);
            if (e) return e;
        }
        return Error();
    }
    // one raw record per non-directory entry; every read goes through the seams and is keyed by
    // info.Name() under basePath exactly like :142,:151,:157,:164
    kxpu_devrec r;
    auto readNuma = [&](std::string &out) { return p.readNumaNode(p.basePath, name, out); };
    std::vector<std::string> allowed;
    Error e = leafRecord(name, p.xpuClasses,
                         [&](const char *prop, std::string &out) { return p.readIDFromFile(p.basePath, name, prop, out); },
                         [&](const char *link, std::string &out) { return p.readLink(p.basePath, name, link, out); },
                         p.readsNuma() ? &readNuma : nullptr, allowedDrivers(p, allowed), r);
    if (e) return e;
    recs.push_back(r);
    if (paths) {  // readsPaths(): the entry's link, one readlink
        kxpu_pcipath pp;
        std::string target;
        if (p.readPciPath(p.basePath, name, target)) pciPathRecord(target, pp);
        else memset(&pp, 0, sizeof pp);
        paths->push_back(pp);
    }
    return Error();
}

Error Plugin::gatherRecords(std::vector<kxpu_devrec> &recs, std::vector<kxpu_pcipath> *paths, std::vector<int64_t> *cdevs,
                            std::vector<kxpu_sriovrec> *srs) {
    recs.clear();
    if (paths) paths->clear();
    size_t slash = basePath.find_last_of('/');
    Error e = walkDir(*this, basePath, slash == std::string::npos ? basePath : basePath.substr(slash + 1), recs,
                      readsPaths() ? paths : nullptr);
    readCdevs(recs, cdevs);
    readSriovs(recs, srs);
    return e;
}

bool Plugin::cdevEnabled() const {
    for (const XpuClass &c : xpuClasses)
        if (c.vfioCdev) return true;
    return false;
}

bool Plugin::mdevCdevEnabled() const {
    for (const XpuClass &c : vgpuClasses)
        if (c.mdevCdev) return true;
    return false;
}

int64_t Plugin::readVfioCdev(const std::string &base, const std::string &entry) {
    cdevReads++;
    DIR *d = opendir((base + "/" + entry + "/vfio-dev").c_str());
    if (!d) return -1;
    std::string node;
    int entries = 0;
    while (struct dirent *de = readdir(d)) {
        if (strcmp(de->d_name, ".") == 0 || strcmp(de->d_name, "..") == 0) continue;
        if (++entries == 1) node = de->d_name;
    }
    closedir(d);
    if (entries != 1 || node.size() < 5 || node.size() > 14 || node.compare(0, 4, "vfio") != 0) return -1;
    const std::string num = node.substr(4);
    if (num.size() > 1 && num[0] == '0') return -1;  // canonical decimals only
    uint64_t v = 0;
    for (char ch : num) {
        if (ch < '0' || ch > '9') return -1;
        v = v * 10 + (uint64_t)(ch - '0');
    }
    return v < (1ull << 32) ? (int64_t)v : -1;
}

// does a record with this vendor and driver match a class that sets `flag` (vfioCdev or mdevCdev; nullptr: any class)?
template <typename Rec>
static bool cdevClassOf(const std::vector<XpuClass> &classes, bool XpuClass::*flag, const Rec &r, const uint8_t *vendorTxt,
                        size_t vendorCap) {
    if (r.flags & (KXPU_REC_IS_DIR | KXPU_REC_VENDOR_ERR | KXPU_REC_DRIVER_ERR)) return false;
    const std::string vendor = trimID(std::string((const char *)vendorTxt, std::min<size_t>(r.vendor_len, vendorCap)));
    const std::string drv(r.driver, strnlen(r.driver, sizeof r.driver));
    bool match = false;
    for (const XpuClass &c : classes) match |= (!flag || c.*flag) && c.vendor == vendor && c.driver == drv;
    return match;
}

// the vfio-dev/ read of every record that matches a vfioCdev class (vendor and driver), after either gather
void Plugin::readCdevs(const std::vector<kxpu_devrec> &recs, std::vector<int64_t> *cdevs) {
    if (!cdevs) return;
    cdevs->clear();
    if (!cdevEnabled()) return;
    cdevs->assign(recs.size(), -1);
    for (size_t i = 0; i < recs.size(); i++) {
        const kxpu_devrec &r = recs[i];
        if (cdevClassOf(xpuClasses, &XpuClass::vfioCdev, r, r.vendor_txt, sizeof r.vendor_txt))
            (*cdevs)[i] = readVfioCdev(basePath, std::string(r.bdf, strnlen(r.bdf, sizeof r.bdf)));
    }
}

kxpu_sriovrec Plugin::readSriov(const std::string &bdf) {
    sriovReads++;
    kxpu_sriovrec s;
    memset(&s, 0, sizeof s);
    const std::string dir = basePath + "/" + bdf + "/";
    char buf[4096];
    const ssize_t n = readlink((dir + "physfn").c_str(), buf, sizeof buf - 1);
    if (n >= 0) {
        const std::string target(buf, (size_t)n);
        const size_t slash = target.find_last_of('/');
        const std::string pf = slash == std::string::npos ? target : target.substr(slash + 1);
        if (pf.size() < sizeof s.physfn) memcpy(s.physfn, pf.data(), pf.size());
        else s.flags |= KXPU_SR_PHYSFN_ERR;  // no PCI address is this long
    } else if (errno != ENOENT) {
        s.flags |= KXPU_SR_PHYSFN_ERR;
    }
    FILE *f = fopen((dir + "sriov_numvfs").c_str(), "rb");
    if (f) {
        uint8_t txt[sizeof s.numvfs_txt + 1];
        const size_t got = fread(txt, 1, sizeof txt, f);
        if (ferror(f)) s.flags |= KXPU_SR_NUMVFS_ERR;
        fclose(f);
        memcpy(s.numvfs_txt, txt, std::min(got, sizeof s.numvfs_txt));
        s.numvfs_len = (uint8_t)got;  // 9: longer than the record holds
    } else if (errno != ENOENT) {
        s.flags |= KXPU_SR_NUMVFS_ERR;
    }
    return s;
}

// the SR-IOV reads of every candidate of a passthrough class, after either gather
void Plugin::readSriovs(const std::vector<kxpu_devrec> &recs, std::vector<kxpu_sriovrec> *srs) {
    if (!srs) return;
    srs->clear();
    if (!sriovAware) return;
    kxpu_sriovrec zero;
    memset(&zero, 0, sizeof zero);
    srs->assign(recs.size(), zero);
    for (size_t i = 0; i < recs.size(); i++) {
        const kxpu_devrec &r = recs[i];
        if (!(r.flags & KXPU_REC_IOMMU_ERR) && cdevClassOf(xpuClasses, nullptr, r, r.vendor_txt, sizeof r.vendor_txt))
            (*srs)[i] = readSriov(std::string(r.bdf, strnlen(r.bdf, sizeof r.bdf)));
    }
}

static bool isClassDriver(const std::vector<XpuClass> &classes, const std::string &driver);

void Plugin::readResets(std::vector<kxpu_devrec> &recs, std::vector<kxpu_resetrec> &rrs) {
    rrs.clear();
    if (!resetCheck) return;
    kxpu_resetrec zero;
    memset(&zero, 0, sizeof zero);
    rrs.assign(recs.size(), zero);
    for (size_t i = 0; i < recs.size(); i++) {
        kxpu_devrec &r = recs[i];
        if (r.flags & KXPU_REC_IS_DIR) continue;
        const std::string bdf(r.bdf, strnlen(r.bdf, sizeof r.bdf));
        std::string s;
        if (!r.driver[0] && !(r.flags & KXPU_REC_DRIVER_ERR) && readLink(basePath, bdf, "driver", s))  // the class test
            memcpy(r.driver, s.data(), std::min(s.size(), sizeof r.driver - 1));  // did not need it: bus-reset sets do
        const std::string drv(r.driver, strnlen(r.driver, sizeof r.driver));
        const bool candidate = cdevClassOf(xpuClasses, nullptr, r, r.vendor_txt, sizeof r.vendor_txt);
        if (!candidate && !(r.flags & KXPU_REC_BLOCKS) && isClassDriver(xpuClasses, drv)) {  // its group is not known yet
            uint32_t g = 0;
            if (readLink(basePath, bdf, "iommu_group", s) && parseGroup(s, g)) r.iommu_group = g;
            else r.flags |= KXPU_REC_IOMMU_ERR;
        }
        if (!candidate || (r.flags & KXPU_REC_IOMMU_ERR)) continue;
        kxpu_resetrec &rr = rrs[i];
        resetReads++;
        if (readResetFile(basePath, bdf, "reset_method", s)) {
            memcpy(rr.txt, s.data(), std::min(s.size(), sizeof rr.txt));
            rr.len = (uint8_t)std::min<size_t>(s.size(), sizeof rr.txt + 1);
        } else if (errno != ENOENT) {
            rr.flags |= KXPU_RS_READ_ERR;
        } else {
            rr.flags |= KXPU_RS_ABSENT;
            resetReads++;
            if (readResetFile(basePath, bdf, "reset", s)) rr.flags |= KXPU_RS_LEGACY;
        }
    }
}

bool Plugin::vfVgpuEnabled() const {
    for (const XpuClass &c : xpuClasses)
        if (c.vfVgpu) return true;
    return false;
}

bool Plugin::passthroughDriver(const std::string &driver) const {
    for (const XpuClass &c : xpuClasses)
        if (!c.vfVgpu && c.driver == driver) return true;
    return false;
}

// current_vgpu_type of <basePath>/<bdf> into a side record marked read; counts in vfVgpuReads
static void readCurrentType(Plugin &p, const std::string &bdf, kxpu_vfvgpurec &v) {
    v.flags = KXPU_VT_READ;
    std::string cur;
    p.vfVgpuReads++;
    if (p.readVgpuFile(p.basePath, bdf, "current_vgpu_type", cur)) {
        memcpy(v.cur_txt, cur.data(), std::min(cur.size(), sizeof v.cur_txt));
        v.cur_len = (uint8_t)std::min<size_t>(cur.size(), sizeof v.cur_txt + 1);
    } else {
        v.flags |= KXPU_VT_CUR_ERR;
    }
}

// vfVgpu: current_vgpu_type and creatable_vgpu_types of every VF (a record with a physfn link) of such a class; with
// vfVgpuDraEnabled or vfVgpuHealth also the basename of that link
void Plugin::readVfVgpus(PciWalk &w) {
    w.vts.clear();
    w.creatable.clear();
    w.physfn.clear();
    if (!vfVgpuEnabled()) return;
    kxpu_vfvgpurec zero;
    memset(&zero, 0, sizeof zero);
    w.vts.assign(w.recs.size(), zero);
    w.creatable.assign(w.recs.size(), std::string());
    if (vfVgpuDraEnabled() || vfVgpuHealth) w.physfn.assign(w.recs.size(), std::string());
    for (size_t i = 0; i < w.recs.size(); i++) {
        const kxpu_devrec &r = w.recs[i];
        if (!cdevClassOf(xpuClasses, &XpuClass::vfVgpu, r, r.vendor_txt, sizeof r.vendor_txt)) continue;
        const std::string bdf(r.bdf, strnlen(r.bdf, sizeof r.bdf));
        char buf[256];
        const ssize_t ln = readlink((basePath + "/" + bdf + "/physfn").c_str(), buf, sizeof buf);
        if (ln < 0) continue;  // no VF: the PF
        if (!w.physfn.empty()) {
            const std::string target(buf, (size_t)ln);
            w.physfn[i] = target.substr(target.rfind('/') + 1);
        }
        readCurrentType(*this, bdf, w.vts[i]);
        std::string tab;
        vfVgpuReads++;
        if (readVgpuFile(basePath, bdf, "creatable_vgpu_types", tab)) {
            if (tab.size() > KXPU_VGPU_FILE_MAX)
                fprintf(stderr, "%s: nvidia/creatable_vgpu_types is longer than %d bytes and is not used\n", bdf.c_str(),
                        KXPU_VGPU_FILE_MAX);
            else
                w.creatable[i] = std::move(tab);
        }
    }
}

// kxpu_vf_vgpu_types over the name tables: every vfVgpu class's vgpuTypeNames, the VFs' creatable_vgpu_types in walk
// order, then the types learned by earlier walks.  A NAMED VF's type joins the learned ones.
Error Plugin::joinVgpuTypes(PciWalk &w) {
    const size_t n = w.recs.size();
    std::string blob;
    std::vector<uint64_t> off{0};
    auto table = [&](const std::string &t) { blob += t; off.push_back(blob.size()); };
    for (const XpuClass &c : xpuClasses) {
        if (!c.vfVgpu) continue;
        std::string t;
        for (const auto &kv : c.vgpuTypeNames) t += std::to_string(kv.first) + " : " + kv.second + "\n";
        table(t);
    }
    for (const std::string &t : w.creatable)
        if (!t.empty()) table(t);
    std::string learned;
    for (const auto &kv : learnedVgpuTypes_) learned += std::to_string(kv.first) + " : " + kv.second + "\n";
    table(learned);
    kxpu_vgpukey zero;
    memset(&zero, 0, sizeof zero);
    w.vkeys.assign(n ? n : 1, zero);
    w.vtype.assign(n ? n : 1, 0);
    w.vstatus.assign(n ? n : 1, KXPU_VT_NONE);
    const int32_t rc = kxpu_vf_vgpu_types(ctx_, w.vts.data(), n, (const uint8_t *)blob.data(), off.data(), off.size() - 1,
                                          w.vkeys.data(), w.vtype.data(), w.vstatus.data());
    if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_vf_vgpu_types", rc);
    for (size_t i = 0; i < n; i++) {
        const std::string bdf(w.recs[i].bdf, strnlen(w.recs[i].bdf, sizeof w.recs[i].bdf));
        if (w.vstatus[i] == KXPU_VT_NAMED)
            learnedVgpuTypes_.emplace(w.vtype[i], std::string((const char *)w.vkeys[i].key, w.vkeys[i].len));
        else if (w.vstatus[i] == KXPU_VT_UNNAMED)
            fprintf(stderr, "%s carries vGPU type %u, which no creatable_vgpu_types list or vgpuTypeNames entry names; not served\n",
                    bdf.c_str(), w.vtype[i]);
        else if (w.vstatus[i] == KXPU_VT_BAD)
            fprintf(stderr, "%s: nvidia/current_vgpu_type could not be read or holds no vGPU type ID; not served\n", bdf.c_str());
    }
    return Error();
}

Error Plugin::gatherVfVgpu(PciWalk &w) {
    Error e = gatherRecords(w.recs);
    readVfVgpus(w);
    return e;
}

// vfVgpuHealth without a vfVgpu class; vfVgpu with draDriver, or on a vGPU class, and vgpuDraDriver without vfVgpu:
// refused, naming the class
Error Plugin::checkVfVgpuClasses() const {
    if (vfVgpuHealth && !vfVgpuEnabled()) return fail("vfVgpuHealth is set but no class has vfVgpu");
    for (const XpuClass &c : xpuClasses)
        if (c.vfVgpu && !c.draDriver.empty())
            return fail("class " + c.vendor + "/" + c.driver + " (" + c.cdiKind + "): vfVgpu cannot be published as DRA ResourceSlices (draDriver " + c.draDriver + ")");
    for (const XpuClass &c : vgpuClasses)
        if (c.vfVgpu)
            return fail("vGPU class " + c.vendor + "/" + c.driver + " (" + c.cdiKind + "): vfVgpu applies to passthrough classes only");
    for (const XpuClass &c : xpuClasses)
        if (!c.vfVgpu && !c.vgpuDraDriver.empty())
            return fail("class " + c.vendor + "/" + c.driver + " (" + c.cdiKind + "): vgpuDraDriver " + c.vgpuDraDriver +
                        " needs vfVgpu on the class");
    for (const XpuClass &c : vgpuClasses)
        if (!c.vgpuDraDriver.empty())
            return fail("vGPU class " + c.vendor + "/" + c.driver + " (" + c.cdiKind + "): vgpuDraDriver " + c.vgpuDraDriver +
                        " applies to vfVgpu classes only");
    return Error();
}

// a Kubernetes qualified name (the part after the prefix): 1-63 bytes, alphanumeric at both ends, [-A-Za-z0-9_.] inside
static bool qualifiedName(const std::string &v) {
    auto alnum = [](char ch) { return (ch >= '0' && ch <= '9') || (ch >= 'a' && ch <= 'z') || (ch >= 'A' && ch <= 'Z'); };
    if (v.empty() || v.size() > 63 || !alnum(v.front()) || !alnum(v.back())) return false;
    for (char ch : v)
        if (!alnum(ch) && ch != '-' && ch != '_' && ch != '.') return false;
    return true;
}

// draPcieDomain (kxpu_dra_slices_pcie's attr_domain): empty, or a lowercase DNS subdomain of at most 63 bytes that is
// neither kubernetes.io nor k8s.io nor under either, and only with a passthrough class that has a draDriver
Error Plugin::checkDraPcieDomain() const {
    const std::string &d = draPcieDomain;
    if (d.empty()) return Error();
    const std::string what = "draPcieDomain \"" + d + "\"";
    bool ok = d.size() <= 63;
    for (size_t start = 0; ok && start <= d.size();) {
        size_t end = d.find('.', start);
        if (end == std::string::npos) end = d.size();
        auto lower = [](char ch) { return (ch >= '0' && ch <= '9') || (ch >= 'a' && ch <= 'z'); };
        ok = end > start && end - start <= 63 && lower(d[start]) && lower(d[end - 1]);
        for (size_t i = start; ok && i < end; i++) ok = lower(d[i]) || d[i] == '-';
        start = end + 1;
    }
    if (!ok) return fail(what + " is not a lowercase DNS subdomain of at most 63 bytes");
    for (const char *reserved : {"kubernetes.io", "k8s.io"}) {
        const std::string r(reserved);
        if (d == r || (d.size() > r.size() && d.compare(d.size() - r.size() - 1, std::string::npos, "." + r) == 0))
            return fail(what + " is reserved: names under " + r + " are the standard attributes'");
    }
    if (!draEnabled()) return fail(what + " is set but no passthrough class has a draDriver");
    return Error();
}

// draVgpuPcie: the vGPU pools' attributes take draPcieDomain's names, and only a vGPU class with DRA publishes them
Error Plugin::checkDraVgpuPcie() const {
    if (!draVgpuPcie) return Error();
    if (draPcieDomain.empty()) return fail("draVgpuPcie is set but draPcieDomain is empty: it names the attributes");
    if (!vgpuDraEnabled() && !vfVgpuDraEnabled())
        return fail("draVgpuPcie is set but no vGPU class publishes DRA (no vGPU class has a draDriver, no class a vgpuDraDriver)");
    return Error();
}

Error Plugin::checkResourceNames() const {
    size_t total = 0;
    std::map<std::string, size_t> classOf;  // name -> the class that configures it
    for (size_t k = 0; k < xpuClasses.size(); k++) {
        const XpuClass &c = xpuClasses[k];
        const std::string cls = "class " + c.vendor + "/" + c.driver + " (" + c.cdiKind + ")";
        if (c.resourceNames.empty()) continue;
        if (c.vfVgpu) return fail(cls + ": resourceNames cannot rename a vfVgpu class, whose vGPUs are named by their type keys");
        for (const auto &kv : c.resourceNames) {
            bool hex = kv.first.size() == 4;
            for (char ch : kv.first) hex = hex && ((ch >= '0' && ch <= '9') || (ch >= 'a' && ch <= 'f'));
            if (!hex && kv.first != "*")
                return fail(cls + ": resourceNames key \"" + kv.first + "\" is neither 4 lowercase hex digits nor \"*\"");
            if (!qualifiedName(kv.second))
                return fail(cls + ": resourceNames[\"" + kv.first + "\"] = \"" + kv.second +
                            "\" is not a qualified name (1-63 bytes, alphanumeric at both ends, [-A-Za-z0-9_.] inside)");
            auto it = classOf.find(kv.second);
            if (it != classOf.end() && it->second != k)
                return fail(cls + ": resourceNames[\"" + kv.first + "\"] = \"" + kv.second + "\" is also configured on class " +
                            xpuClasses[it->second].vendor + "/" + xpuClasses[it->second].driver + " (" +
                            xpuClasses[it->second].cdiKind + "); socket names ignore the namespace");
            classOf.emplace(kv.second, k);
        }
        total += c.resourceNames.size();
        if (total > KXPU_MAX_NAMES)
            return fail(cls + ": resourceNames brings the entries of all classes to " + std::to_string(total) + ", over " +
                        std::to_string(KXPU_MAX_NAMES));
    }
    for (const XpuClass &c : vgpuClasses)
        if (!c.resourceNames.empty())
            return fail("vGPU class " + c.vendor + "/" + c.driver + " (" + c.cdiKind +
                        "): resourceNames cannot rename a vGPU class, whose vGPUs are named by their type keys");
    return Error();
}

void Plugin::nameTable(std::vector<kxpu_name_entry> &entries, std::vector<std::string> &slotNames) const {
    entries.clear();
    slotNames.clear();
    for (size_t k = 0; k < xpuClasses.size(); k++) {
        std::map<std::string, uint32_t> slotOf;  // this class's names
        for (const auto &kv : xpuClasses[k].resourceNames) {
            auto it = slotOf.find(kv.second);
            if (it == slotOf.end()) {
                it = slotOf.emplace(kv.second, (uint32_t)slotNames.size()).first;
                slotNames.push_back(kv.second);
            }
            kxpu_name_entry e;
            memset(&e, 0, sizeof e);
            e.rule = (uint32_t)k;
            e.slot = it->second;
            memcpy(e.device, kv.first.data(), std::min(kv.first.size(), sizeof e.device));
            entries.push_back(e);
        }
    }
}

// ---------------------------------------------------------------------------- SURVEY 8(f) row 2
// Batched sysfs ingestion: the same records as gatherRecords, but the entries of basePath are read
// with paths RELATIVE to one directory descriptor (openat / readlinkat on "<bdf>/vendor": no lstat per
// entry -- getdents64 already says what is a directory --, no absolute path resolution, no FILE
// buffering) and by several threads, each filling its own slice of the record table, so that S1 ends
// in one contiguous table ready for a single H2D copy.  Only with the default seams; real directories
// under basePath (never on sysfs) go through the generic walk at their position.
Error Plugin::gatherRecordsFast(std::vector<kxpu_devrec> &recs, unsigned threads, std::vector<kxpu_pcipath> *paths,
                                std::vector<int64_t> *cdevs, std::vector<kxpu_sriovrec> *srs) {
    Error e = gatherRecordsFastWalk(recs, threads, paths);
    readCdevs(recs, cdevs);
    readSriovs(recs, srs);
    return e;
}

Error Plugin::gatherRecordsFastWalk(std::vector<kxpu_devrec> &recs, unsigned threads, std::vector<kxpu_pcipath> *paths) {
    recs.clear();
    if (paths) paths->clear();
    if (!readsPaths()) paths = nullptr;
    struct stat sb;
    if (lstat(basePath.c_str(), &sb) != 0) return fail("Error accessing file path \"" + basePath + "\": " + strerror(errno));
    // the fast reads bypass the seams: only when nobody replaced them (tests do, device_plugin.go:38-39)
    using SeamFn = bool (*)(const std::string &, const std::string &, const std::string &, std::string &);
    SeamFn const *rl = readLink.target<SeamFn>(), *ri = readIDFromFile.target<SeamFn>();
    using NumaFn = bool (*)(const std::string &, const std::string &, std::string &);
    NumaFn const *rn = readNumaNode.target<NumaFn>();
    NumaFn const *rp = readPciPath.target<NumaFn>();
    const bool defaultSeams = rl && *rl == readLinkFunc && ri && *ri == readIDFromFileFunc &&
                              (!readsNuma() || (rn && *rn == readNumaNodeFunc)) &&
                              (!paths || (rp && *rp == readPciPathFunc));
    if (!S_ISDIR(sb.st_mode) || !defaultSeams) return gatherRecords(recs, paths);
    int basefd = open(basePath.c_str(), O_RDONLY | O_DIRECTORY | O_CLOEXEC);
    if (basefd < 0) return fail("Error accessing file path \"" + basePath + "\": " + strerror(errno));
    DIR *d = fdopendir(dup(basefd));
    if (!d) { close(basefd); return fail("Error accessing file path \"" + basePath + "\": " + strerror(errno)); }
    struct Ent { std::string name; bool dir; };
    std::vector<Ent> ents;
    while (struct dirent *de = readdir(d)) {
        if (strcmp(de->d_name, ".") == 0 || strcmp(de->d_name, "..") == 0) continue;
        bool isdir = de->d_type == DT_DIR;
        if (de->d_type == DT_UNKNOWN) {  // file systems without d_type: one fstatat, still no path walk
            struct stat es;
            isdir = fstatat(basefd, de->d_name, &es, AT_SYMLINK_NOFOLLOW) == 0 && S_ISDIR(es.st_mode);
        }
        ents.push_back(Ent{de->d_name, isdir});
    }
    closedir(d);
    std::sort(ents.begin(), ents.end(), [](const Ent &a, const Ent &b) { return a.name < b.name; });

    const size_t N = ents.size();
    std::vector<kxpu_devrec> flat(N);
    std::vector<kxpu_pcipath> flatPaths(paths ? N : 0);
    std::vector<Error> errs(N);
    std::vector<std::string> allowedBuf;
    const std::vector<std::string> *allowed = allowedDrivers(*this, allowedBuf);
    auto readID = [&](const std::string &name, const char *prop, std::string &out) {
        const std::string rel = name + "/" + prop;
        int fd = openat(basefd, rel.c_str(), O_RDONLY | O_CLOEXEC);
        if (fd < 0) {
            fprintf(stderr, "Could not read %s for device %s: %s\n", prop, name.c_str(), strerror(errno));
            return false;
        }
        char buf[256];
        size_t got = 0;
        for (;;) {  // os.ReadFile reads to EOF
            ssize_t k = read(fd, buf + got, sizeof buf - got);
            if (k < 0) { close(fd); return false; }
            if (k == 0) break;
            got += (size_t)k;
            if (got == sizeof buf) break;
        }
        close(fd);
        out.assign(buf, got);
        return true;
    };
    auto readLnk = [&](const std::string &name, const char *link, std::string &out) {
        const std::string rel = name + "/" + link;
        char buf[4096];
        ssize_t k = readlinkat(basefd, rel.c_str(), buf, sizeof buf - 1);
        if (k < 0) {
            fprintf(stderr, "Could not read link %s for device %s: %s\n", link, name.c_str(), strerror(errno));
            return false;
        }
        std::string target(buf, (size_t)k);
        size_t slash = target.find_last_of('/');
        out = slash == std::string::npos ? target : target.substr(slash + 1);
        return true;
    };
    auto work = [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; i++) {
            if (ents[i].dir) continue;
            const std::string &name = ents[i].name;
            // numa_node on the same directory descriptor; quiet like readNumaNodeFunc
            auto readNuma = [&](std::string &out) {
                int fd = openat(basefd, (name + "/numa_node").c_str(), O_RDONLY | O_CLOEXEC);
                if (fd < 0) return false;
                char buf[64];
                ssize_t k = read(fd, buf, sizeof buf);
                close(fd);
                if (k < 0) return false;
                out.assign(buf, (size_t)k);
                return true;
            };
            errs[i] = leafRecord(name, xpuClasses, [&](const char *prop, std::string &out) { return readID(name, prop, out); },
                                 [&](const char *link, std::string &out) { return readLnk(name, link, out); },
                                 readsNuma() ? &readNuma : nullptr, allowed, flat[i]);
            if (paths && !errs[i]) {  // the entry's own link on the same directory descriptor
                char buf[4096];
                const ssize_t k = readlinkat(basefd, name.c_str(), buf, sizeof buf);
                if (k >= 0 && k < (ssize_t)sizeof buf) pciPathRecord(std::string(buf, (size_t)k), flatPaths[i]);
                else memset(&flatPaths[i], 0, sizeof flatPaths[i]);
            }
        }
    };
    if (threads == 0) threads = std::min(8u, std::max(1u, std::thread::hardware_concurrency()));
    threads = (unsigned)std::min<size_t>(threads, std::max<size_t>(N / 64, 1));
    if (threads <= 1) {
        work(0, N);
    } else {
        std::vector<std::thread> pool;
        for (unsigned t = 0; t < threads; t++) pool.emplace_back(work, N * t / threads, N * (t + 1) / threads);
        for (auto &th : pool) th.join();
    }
    close(basefd);
    // assemble in walk order; the first error in walk order wins, like the sequential walk
    for (size_t i = 0; i < N; i++) {
        if (ents[i].dir) {
            Error e = walkDir(*this, basePath + "/" + ents[i].name, ents[i].name, recs, paths);
            if (e) return e;
        } else {
            if (errs[i]) return errs[i];
            recs.push_back(flat[i]);
            if (paths) paths->push_back(flatPaths[i]);
        }
    }
    return Error();
}

static std::string devIdString(uint64_t packed) {
    char b[9];
    memcpy(b, &packed, 8);
    b[8] = 0;
    return std::string(b);
}

// mdevCdev names an mdev's cdev: a passthrough class with it is refused
static Error checkPassthroughClasses(const std::vector<XpuClass> &classes) {
    for (const XpuClass &c : classes)
        if (c.mdevCdev)
            return fail("passthrough class " + c.vendor + "/" + c.driver + " (" + c.cdiKind + "): mdevCdev applies to vGPU classes only; a passthrough class sets vfioCdev");
    return Error();
}

// the parse calls of the PCI resume into the record type of the passthrough spec paths (cdiRecord): the untyped layouts
// give type_id 0
template <int32_t (*parse)(kxpu_ctx *, int32_t, const char *, const uint8_t *, size_t, kxpu_cdidev *, size_t, size_t *)>
static int32_t parseUntyped(kxpu_ctx *ctx, int32_t fmt, const char *kind, const uint8_t *doc, size_t len, kxpu_vfvgpucdi *out,
                            size_t cap, size_t *n) {
    std::vector<kxpu_cdidev> d(cap);
    const int32_t rc = parse(ctx, fmt, kind, doc, len, d.data(), cap, n);
    if (rc == KXPU_OK)
        for (size_t i = 0; i < *n; i++) {
            memset(&out[i], 0, sizeof out[i]);
            out[i].dev = d[i];
        }
    return rc;
}
static int32_t parsePciGroup(kxpu_ctx *ctx, int32_t fmt, const char *kind, const uint8_t *doc, size_t len, kxpu_vfvgpucdi *out,
                             size_t cap, size_t *n) {
    return parseUntyped<kxpu_cdi_parse>(ctx, fmt, kind, doc, len, out, cap, n);
}
static int32_t parsePciCdev(kxpu_ctx *ctx, int32_t fmt, const char *kind, const uint8_t *doc, size_t len, kxpu_vfvgpucdi *out,
                            size_t cap, size_t *n) {
    return parseUntyped<kxpu_cdi_parse_cdev>(ctx, fmt, kind, doc, len, out, cap, n);
}

// createIommuDeviceMap, device_plugin.go:126-180
Error Plugin::createIommuDeviceMap() {
    {
        Error e = checkPassthroughClasses(xpuClasses);
        if (e) return e;
    }
    iommuMap.clear();   // :127
    deviceMap.clear();  // :128
    iommuState.clear();
    deviceClass.clear();
    deviceNamed.clear();
    // the generation is read BEFORE the walk: an event during the walk makes the snapshot stale, never fresh
    pci_.haveGen = bindGeneration && bindGeneration(pci_.gen);
    haveSnapshotGen_ = snapshotValidation && pci_.haveGen;
    snapshotGen_ = pci_.gen;
    PciWalk w;
    std::vector<kxpu_snaprec> prev;
    uint64_t next = 0;
    if (resumeIndices) {  // the previous specs before the walk: a typed spec names the vGPU types of the VFs it lists
        resume_ = ResumeReport();  // the mdev walk resumes from the same report and state file
        readIndexState();
        previousEntries<kxpu_vfvgpucdi>(xpuClasses, parsePciGroup, resume_.stateRead ? resume_.statePci : 0, resume_.pci,
                                        prev, next);
    }
    Error e = firstWalk(w, pci_);
    if (e || !resumeIndices) return e;
    return resume(w, pci_, resume_.pci, resume_.stateRead ? resume_.statePci : 0, std::move(prev), next);
}

template <typename Walk>
Error Plugin::firstWalk(Walk &w, WalkBook &book) {
    Error e = classify(w);
    if (e) return e;
    buildMaps(w, nullptr);
    book.snap = snapshotOf(w, nullptr);  // host bookkeeping for a later rediscovery: no GPU call
    book.next = book.snap.size();
    return Error();
}

// one rule per class: rule index == class index
static std::vector<kxpu_xpu_rule> classRules(const std::vector<XpuClass> &classes) {
    std::vector<kxpu_xpu_rule> rules(classes.size());
    for (size_t c = 0; c < classes.size(); c++) {
        kxpu_xpu_rule &r = rules[c];
        const char *vendor = classes[c].vendor.c_str(), *driver = classes[c].driver.c_str();
        memset(&r, 0, sizeof r);  // NUL padded; a field filled to its end is left for kxpu_classify_rules to reject
        memcpy(r.vendor, vendor, strnlen(vendor, sizeof r.vendor));
        memcpy(r.driver, driver, strnlen(driver, sizeof r.driver));
    }
    return rules;
}

kxpu_classify_out ClassifyResult::wire(size_t n) {
    accept.assign(n, 0); gids.assign(n, 0); goff.assign(n + 1, 0); gmem.assign(n, 0); doff.assign(n + 1, 0);
    dgrp.assign(n, 0); dids.assign(n, 0);
    drule.assign(n ? n : 1, 0);
    gnuma.assign(n ? n : 1, 0);
    kxpu_classify_out out;
    memset(&out, 0, sizeof out);
    out.accept_index = accept.data(); out.group_ids = gids.data(); out.group_off = goff.data();
    out.group_members = gmem.data(); out.dev_ids = dids.data(); out.dev_off = doff.data(); out.dev_groups = dgrp.data();
    return out;
}

// class of a group = the rule of its first member, which the device-map entry listing it carries
static std::map<uint32_t, size_t> groupClasses(const ClassifyResult &r) {
    std::map<uint32_t, size_t> groupClass;
    for (uint32_t d = 0; d < r.nDevids; d++)
        for (uint32_t k = r.doff[d]; k < r.doff[d + 1]; k++) groupClass[r.dgrp[k]] = r.drule[d];
    return groupClass;
}

// the class an accepted record itself matched (a group may hold records of several classes): the class of its
// (vendor, driver) pair
static size_t recordClass(const std::vector<XpuClass> &classes, const uint8_t *vendorTxt, uint8_t vendorLen, const char *driver,
                          size_t driverCap) {
    const std::string vendor = trimID(std::string((const char *)vendorTxt, vendorLen));
    const std::string drv(driver, strnlen(driver, driverCap));
    size_t cls = 0;
    for (size_t c = 0; c < classes.size(); c++)
        if (classes[c].vendor == vendor && classes[c].driver == drv) cls = c;
    return cls;
}

// "<bdf> is bound to <driver>" of a blocking record
static std::string blockerOf(const kxpu_devrec &r) {
    return std::string(r.bdf, strnlen(r.bdf, sizeof r.bdf)) + " is bound to " + std::string(r.driver, strnlen(r.driver, sizeof r.driver));
}

// the PCIe root of a kxpu_pcipath: its first component when that is "pci" followed by 1..13 bytes of [0-9a-f:]; "" for
// anything else (unknown)
static std::string pcieRootOf(const kxpu_pcipath *path) {
    if (!path || path->len == 0 || path->len > sizeof path->path) return std::string();
    const std::string p(path->path, path->len);
    const std::string root = p.substr(0, p.find('/'));
    bool ok = root.size() >= 4 && root.size() <= sizeof(kxpu_dradev::pcie_root) && root.compare(0, 3, "pci") == 0;
    for (size_t k = 3; ok && k < root.size(); k++)
        ok = (root[k] >= '0' && root[k] <= '9') || (root[k] >= 'a' && root[k] <= 'f') || root[k] == ':';
    return ok ? root : std::string();
}

// the ResourceSlice record of a group (product left empty): bdf, vendor and device of its first member r, the PCIe root
// of r's path (pcieRootOf), and the group's NUMA mask
static kxpu_dradev draRecord(const kxpu_devrec &r, const kxpu_pcipath *path, uint64_t numa) {
    kxpu_dradev d;
    memset(&d, 0, sizeof d);
    memcpy(d.bdf, r.bdf, strnlen(r.bdf, sizeof r.bdf));
    const std::string vendor = trimID(std::string((const char *)r.vendor_txt, std::min<size_t>(r.vendor_len, sizeof r.vendor_txt)));
    const std::string device = trimID(std::string((const char *)r.device_txt, std::min<size_t>(r.device_len, sizeof r.device_txt)));
    memcpy(d.vendor, vendor.data(), std::min(vendor.size(), sizeof d.vendor));
    memcpy(d.device, device.data(), std::min(device.size(), sizeof d.device));
    const std::string root = pcieRootOf(path);
    memcpy(d.pcie_root, root.data(), root.size());
    d.numa_mask = numa;
    d.iommu_group = r.iommu_group;
    return d;
}

static bool isClassDriver(const std::vector<XpuClass> &classes, const std::string &driver) {
    for (const XpuClass &c : classes)
        if (c.driver == driver) return true;
    return false;
}

static std::string sriovVfReason(const std::string &vf, const std::string &pf, const std::string &driver) {
    return vf + " needs the VF token of " + pf + " (bound to " + driver + ")";
}
static std::string sriovPfReason(const std::string &pf, uint32_t numvfs) {
    return pf + " has " + std::to_string(numvfs) + " VFs enabled";
}

// the reason kxpu_sriov blocked on record i of a walk: a VF whose PF is bound to a class driver, else a PF with VFs
// classes: the passthrough classes (a vfVgpu class's driver is the vGPU manager's, which needs no VF token)
static std::string sriovReasonOf(const std::vector<XpuClass> &classes, const PciWalk &w, uint32_t i) {
    const kxpu_devrec &r = w.recs[i];
    const std::string me(r.bdf, strnlen(r.bdf, sizeof r.bdf));
    if (w.pfOf[i] != KXPU_NO_PF) {
        const kxpu_devrec &pf = w.recs[w.pfOf[i]];
        const std::string drv(pf.driver, strnlen(pf.driver, sizeof pf.driver));
        if (!(pf.flags & KXPU_REC_DRIVER_ERR) && isClassDriver(classes, drv))
            return sriovVfReason(me, std::string(pf.bdf, strnlen(pf.bdf, sizeof pf.bdf)), drv);
    }
    return sriovPfReason(me, w.numvfs[i]);
}

static const char *const kResetMethods[7] = {"flr", "af_flr", "pm", "bus", "cxl_bus", "device_specific", "acpi"};

// resetMethods as KXPU_RM_* bits (checkResetMethods refused every other name)
uint32_t Plugin::resetAllow() const {
    uint32_t allow = 0;
    for (const std::string &m : resetMethods)
        for (uint32_t k = 0; k < 7; k++)
            if (m == kResetMethods[k]) allow |= 1u << k;
    return allow;
}

Error Plugin::checkResetMethods() const {
    std::set<std::string> seen;
    for (const std::string &m : resetMethods) {
        if (std::find(std::begin(kResetMethods), std::end(kResetMethods), m) == std::end(kResetMethods))
            return fail("resetMethods: " + m + " is not a reset method (flr, af_flr, pm, bus, cxl_bus, device_specific, acpi)");
        if (!seen.insert(m).second) return fail("resetMethods: " + m + " is listed twice");
    }
    return Error();
}

// why kxpu_reset_check found record i of a walk without a reset: the methods it has that resetMethods does not accept,
// else the function that keeps its bus-reset set from being closed
std::string Plugin::resetReasonOf(const PciWalk &w, uint32_t i) const {
    const std::string me(w.recs[i].bdf, strnlen(w.recs[i].bdf, sizeof w.recs[i].bdf));
    const uint8_t m = w.rmeth[i];
    if (m & KXPU_RM_UNNAMED) return me + " has no reset method in resetMethods (reset: some method, name unknown)";
    if (m) {
        std::string names;
        for (uint32_t k = 0; k < 7; k++)
            if (m & (1u << k)) names += (names.empty() ? "" : " ") + std::string(kResetMethods[k]);
        return me + " has no reset method in resetMethods (reset_method: " + names + ")";
    }
    const uint32_t v = w.rset[i];
    if (v == KXPU_RESET_ROOT_BUS) return me + " has no function reset and sits on a root bus";
    if (v == KXPU_RESET_NO_PATH) return me + " has no function reset and its PCIe path is unknown";
    const kxpu_devrec &r = w.recs[v];
    const std::string other(r.bdf, strnlen(r.bdf, sizeof r.bdf)), drv(r.driver, strnlen(r.driver, sizeof r.driver));
    std::string why;
    if (drv.empty() || (r.flags & KXPU_REC_DRIVER_ERR)) why = "is not bound to a driver";
    else if (!isClassDriver(xpuClasses, drv)) why = "is bound to " + drv;
    else if (r.flags & KXPU_REC_IOMMU_ERR) why = "has no IOMMU group";
    else why = "is in IOMMU group " + std::to_string(r.iommu_group);
    return me + " has no function reset and " + other + " on its bus " + why;  // v != i: a member is class-bound
}

// the walk and classify of createIommuDeviceMap
Error Plugin::classify(PciWalk &w) {
    Error e = gatherRecordsFast(w.recs, 0, &w.paths, &w.cdevs, &w.srs);  // same records as gatherRecords (falls back to it when a seam was replaced)
    if (e) { fprintf(stderr, "%s\n", e.message.c_str()); }  // Walk's error is ignored by the reference (:132)
    readResets(w.recs, w.rrs);
    if (vgpuSriovAware) pciRecs_ = w.recs;  // the mdev walk that follows joins its parents' PFs against them
    const std::vector<kxpu_devrec> &recs = w.recs;
    const size_t n = recs.size();
    ClassifyResult &c = w.out;
    kxpu_classify_out out = c.wire(n);
    const std::vector<kxpu_xpu_rule> rules = classRules(xpuClasses);
    // fatal on failure: there is no CPU path
    int32_t rc;
    const char *what;
    readVfVgpus(w);
    uint32_t vgpuRules = 0;  // vfVgpu: bit r = class r serves vGPU types
    for (size_t k = 0; k < xpuClasses.size(); k++)
        if (xpuClasses[k].vfVgpu) vgpuRules |= 1u << k;
    std::vector<kxpu_name_entry> names;
    std::vector<std::string> slotNames;
    nameTable(names, slotNames);
    c.dslot.clear();
    if (!names.empty()) {  // some class has resourceNames: the same call with the name table
        if (vgpuRules) {
            Error je = joinVgpuTypes(w);
            if (je) return je;
        }
        if (groupViability) c.gblk.assign(n ? n : 1, KXPU_VIABLE);
        c.dslot.assign(n ? n : 1, KXPU_NO_SLOT);
        rc = kxpu_classify_named(ctx_, rules.data(), rules.size(), vgpuRules, recs.data(), n,
                                 vgpuRules ? w.vkeys.data() : nullptr, names.data(), names.size(), &out, c.drule.data(),
                                 c.dslot.data(), readsNuma() ? c.gnuma.data() : nullptr,
                                 groupViability ? c.gblk.data() : nullptr);
        what = "kxpu_classify_named";
    } else if (vgpuRules) {
        Error je = joinVgpuTypes(w);
        if (je) return je;
        if (groupViability) c.gblk.assign(n ? n : 1, KXPU_VIABLE);
        rc = kxpu_classify_vf_vgpu(ctx_, rules.data(), rules.size(), vgpuRules, recs.data(), n, w.vkeys.data(), &out,
                                   c.drule.data(), readsNuma() ? c.gnuma.data() : nullptr,
                                   groupViability ? c.gblk.data() : nullptr);
        what = "kxpu_classify_vf_vgpu";
    } else if (groupViability) {
        c.gblk.assign(n ? n : 1, KXPU_VIABLE);
        rc = kxpu_classify_viable(ctx_, rules.data(), rules.size(), recs.data(), n, &out, c.drule.data(),
                                  readsNuma() ? c.gnuma.data() : nullptr, c.gblk.data());
        what = "kxpu_classify_viable";
    } else {
        rc = readsNuma() ? kxpu_classify_topo(ctx_, rules.data(), rules.size(), recs.data(), n, &out, c.drule.data(), c.gnuma.data())
                         : kxpu_classify_rules(ctx_, rules.data(), rules.size(), recs.data(), n, &out, c.drule.data());
        what = readsNuma() ? "kxpu_classify_topo" : "kxpu_classify_rules";
    }
    if (rc != KXPU_OK) return kxfail(ctx_, what, rc);
    c.nGroups = out.n_groups;
    c.nDevids = out.n_devids;
    if (groupViability)
        for (uint32_t g = 0; g < c.nGroups; g++)
            if (c.gblk[g] != KXPU_VIABLE)
                fprintf(stderr, "IOMMU group %u is not viable: %s\n", c.gids[g], blockerOf(recs[c.gblk[g]]).c_str());
    // the rules of the classes passed through whole: a vfVgpu class's VFs sit on the vGPU manager's driver and need no VF
    // token, so its rule takes no part in the verdict; with none left there is no call
    std::vector<XpuClass> whole;
    for (const XpuClass &k : xpuClasses)
        if (!k.vfVgpu) whole.push_back(k);
    if (sriovAware) {  // the SR-IOV verdict of every group, on the classify CSR
        w.pfOf.assign(n ? n : 1, KXPU_NO_PF);
        w.numvfs.assign(n ? n : 1, 0);
        w.gsriov.assign(c.nGroups + 1, KXPU_VIABLE);
        const std::vector<kxpu_xpu_rule> srules = vgpuRules ? classRules(whole) : rules;
        if (!srules.empty()) {
            rc = kxpu_sriov(ctx_, srules.data(), srules.size(), recs.data(), w.srs.data(), n, c.gids.data(), c.goff.data(),
                            c.gmem.data(), c.nGroups, w.pfOf.data(), w.numvfs.data(), w.gsriov.data());
            if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_sriov", rc);
        }
        for (uint32_t g = 0; g < c.nGroups; g++)
            if (w.gsriov[g] != KXPU_VIABLE)
                fprintf(stderr, "IOMMU group %u is not served: %s\n", c.gids[g], sriovReasonOf(whole, w, w.gsriov[g]).c_str());
    }
    if (resetCheck) {  // every member's function reset or bus-reset set, on the classify CSR
        w.rmeth.assign(n ? n : 1, 0);
        w.rset.assign(n ? n : 1, KXPU_RESET_SET_OK);
        w.greset.assign(c.nGroups + 1, KXPU_VIABLE);
        rc = kxpu_reset_check(ctx_, rules.data(), rules.size(), recs.data(), w.paths.data(), w.rrs.data(), n, resetAllow(),
                              c.goff.data(), c.gmem.data(), c.nGroups, w.rmeth.data(), w.rset.data(), w.greset.data());
        if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_reset_check", rc);
        for (uint32_t g = 0; g < c.nGroups; g++)
            if (w.greset[g] != KXPU_VIABLE)
                fprintf(stderr, "IOMMU group %u is not served: %s\n", c.gids[g], resetReasonOf(w, w.greset[g]).c_str());
    }
    if (pcieTopologyAware) {  // the forest of the walk, one node per group; sriovAware: VFs below their PF
        const size_t cap = (size_t)KXPU_PCIE_MAX_DEPTH * c.nGroups + 1;
        w.gnode.assign(c.nGroups + 1, KXPU_PCIE_NO_NODE);
        w.nodeKey.assign(cap, 0); w.nodeParent.assign(cap, 0); w.nodeDepth.assign(cap, 0);
        if (sriovAware) {
            rc = kxpu_pcie_tree_sriov(ctx_, recs.data(), w.paths.data(), n, c.goff.data(), c.gmem.data(), c.nGroups,
                                      w.gnode.data(), w.nodeKey.data(), w.nodeParent.data(), w.nodeDepth.data(), &w.nNodes,
                                      w.pfOf.data());
        } else {
            rc = kxpu_pcie_tree(ctx_, recs.data(), w.paths.data(), n, c.goff.data(), c.gmem.data(), c.nGroups, w.gnode.data(),
                                w.nodeKey.data(), w.nodeParent.data(), w.nodeDepth.data(), &w.nNodes);
        }
        if (rc != KXPU_OK) return kxfail(ctx_, sriovAware ? "kxpu_pcie_tree_sriov" : "kxpu_pcie_tree", rc);
    }
    if (!draPcieDomain.empty()) {  // each group's root port and switch, from the paths every DRA walk reads
        w.rootPort.assign(c.nGroups + 1, KXPU_PCIE_NO_KEY);
        w.pcieSwitch.assign(c.nGroups + 1, KXPU_PCIE_NO_KEY);
        rc = kxpu_pcie_ports(ctx_, recs.data(), w.paths.data(), n, c.goff.data(), c.gmem.data(), c.nGroups,
                             w.rootPort.data(), w.pcieSwitch.data());
        if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_pcie_ports", rc);
    }
    if (aerPortHealth) {  // the ports above every record, from the paths read above
        w.aerPortOff.assign(n + 1, 0);
        w.aerPortOf.assign((size_t)KXPU_PCIE_MAX_DEPTH * n + 1, 0);
        w.aerPortKey.assign((size_t)KXPU_PCIE_MAX_DEPTH * n + 1, 0);
        uint32_t nk = 0;
        rc = kxpu_aer_ports(ctx_, recs.data(), w.paths.data(), n, w.aerPortOff.data(), w.aerPortOf.data(),
                            w.aerPortKey.data(), &nk);
        if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_aer_ports", rc);
        w.aerPortOf.resize(w.aerPortOff[n]);
        w.aerPortKey.resize(nk);
    }
    return Error();
}

// the device id of a PF record for kxpu_dradevpf: the record's, else (a PF that is no class candidate, whose id the walk
// left unread) <basePath>/<pf>/device read once per PF into `read`; "" when unknown or outside 0..6 bytes of [0-9a-f]
std::string Plugin::pfDeviceOf(const kxpu_devrec &pf, std::map<std::string, std::string> &read) const {
    const std::string bdf(pf.bdf, strnlen(pf.bdf, sizeof pf.bdf));
    std::string id = (pf.flags & KXPU_REC_DEVICE_ERR) ? std::string()
                     : trimID(std::string((const char *)pf.device_txt, std::min<size_t>(pf.device_len, sizeof pf.device_txt)));
    if (id.empty()) {
        auto it = read.find(bdf);
        if (it == read.end()) {
            std::string raw;
            it = read.emplace(bdf, readIDFromFile(basePath, bdf, "device", raw) ? trimID(raw) : "").first;
        }
        id = it->second;
    }
    bool ok = id.size() <= 6;
    for (char ch : id) ok = ok && ((ch >= '0' && ch <= '9') || (ch >= 'a' && ch <= 'f'));
    return ok ? id : std::string();
}

// the sysfs address of a kxpu_pcie_tree function key: a 4-digit domain, or 5..8 digits above ffff (VMD)
static std::string portAddress(uint64_t key) {
    char b[24];
    const unsigned long long dom = key >> 16;
    snprintf(b, sizeof b, dom <= 0xffff ? "%04llx:%02x:%02x.%u" : "%llx:%02x:%02x.%u", dom, (unsigned)(key >> 8 & 0xff),
             (unsigned)(key >> 3 & 0x1f), (unsigned)(key & 7));
    return b;
}

// aerPortHealth: the ports above group g's members (kxpu_aer_ports' CSR of the walk), member by member, each nearest
// first, each port once, with the function (fn of the member) it was first found above
template <typename Dev>
static std::vector<std::pair<std::string, std::string>> groupPorts(const std::vector<uint32_t> &off,
                                                                   const std::vector<uint32_t> &of,
                                                                   const std::vector<uint64_t> &key, const ClassifyResult &c,
                                                                   uint32_t g, const std::vector<Dev> &devs,
                                                                   std::string Dev::*fn) {
    std::vector<std::pair<std::string, std::string>> out;
    std::vector<uint32_t> seen;
    for (uint32_t k = c.goff[g]; k < c.goff[g + 1]; k++) {
        const uint32_t i = c.gmem[k];
        for (uint32_t p = off[i]; p < off[i + 1]; p++) {
            if (std::find(seen.begin(), seen.end(), of[p]) != seen.end()) continue;
            seen.push_back(of[p]);
            out.emplace_back(portAddress(key[of[p]]), devs[k - c.goff[g]].*fn);
        }
    }
    return out;
}

void Plugin::buildMaps(const PciWalk &w, const std::vector<uint64_t> *index) {
    std::map<std::string, std::string> pfDeviceRead;  // sriovPfAware: PF address -> its device file, read once
    iommuMap.clear();
    deviceMap.clear();
    iommuState.clear();
    deviceClass.clear();
    deviceNamed.clear();
    const ClassifyResult &c = w.out;
    std::map<uint32_t, size_t> groupClass = groupClasses(c);
    for (uint32_t g = 0; g < c.nGroups; g++) {
        std::vector<NvidiaGpuDevice> devs;
        for (uint32_t k = c.goff[g]; k < c.goff[g + 1]; k++) {
            const kxpu_devrec &r = w.recs[c.gmem[k]];
            const uint64_t idx = index ? (*index)[c.accept[c.gmem[k]]] : c.accept[c.gmem[k]];
            devs.push_back(NvidiaGpuDevice{std::string(r.bdf), idx});  // :171-174
            devs.back().xpuClass = recordClass(xpuClasses, r.vendor_txt, r.vendor_len, r.driver, sizeof r.driver);
            if (!w.cdevs.empty()) devs.back().cdev = w.cdevs[c.gmem[k]];
            if (!w.vtype.empty() && xpuClasses[devs.back().xpuClass].vfVgpu) {
                devs.back().vgpuType = w.vtype[c.gmem[k]];
                const kxpu_vgpukey &key = w.vkeys[c.gmem[k]];
                devs.back().vgpuKey.assign((const char *)key.key, key.len);
            }
        }
        GroupState<kxpu_dradev> s;
        s.klass = groupClass[c.gids[g]];
        if (topologyAware) s.numa = c.gnuma[g];
        if (pcieTopologyAware) s.pcieNode = w.gnode[g];
        if (!draPcieDomain.empty()) { s.rootPort = w.rootPort[g]; s.pcieSwitch = w.pcieSwitch[g]; }
        if (groupViability && c.gblk[g] != KXPU_VIABLE) s.blocker = blockerOf(w.recs[c.gblk[g]]);
        if (s.blocker.empty() && xpuClasses[s.klass].vfioCdev)  // a member without a cdev: VFIO cannot open it
            for (const NvidiaGpuDevice &d : devs)
                if (d.cdev < 0) { s.blocker = d.addr + " has no VFIO cdev"; s.blockerKind = KXPU_MR_VFIO_CDEV_MISSING; break; }
        if (sriovAware && w.gsriov[g] != KXPU_VIABLE) {
            std::vector<XpuClass> whole;
            for (const XpuClass &k : xpuClasses)
                if (!k.vfVgpu) whole.push_back(k);
            s.sriov = sriovReasonOf(whole, w, w.gsriov[g]);
            if (s.blocker.empty()) { s.blocker = s.sriov; s.blockerKind = KXPU_MR_SRIOV; }
        }
        if (resetCheck && w.greset[g] != KXPU_VIABLE) {
            s.reset = resetReasonOf(w, w.greset[g]);
            if (s.blocker.empty()) { s.blocker = s.reset; s.blockerKind = KXPU_MR_RESET; }
        }
        if (draEnabled()) {
            const uint32_t first = c.gmem[c.goff[g]];
            s.dra = draRecord(w.recs[first], w.paths.size() > first ? &w.paths[first] : nullptr, c.gnuma[g]);
        }
        if (vfVgpuHealth && xpuClasses[s.klass].vfVgpu && !w.physfn.empty()) s.pf = w.physfn[c.gmem[c.goff[g]]];
        if (sriovPfAware && !xpuClasses[s.klass].vfVgpu && w.pfOf[c.gmem[c.goff[g]]] != KXPU_NO_PF) {
            const kxpu_devrec &pf = w.recs[w.pfOf[c.gmem[c.goff[g]]]];
            s.pf.assign(pf.bdf, strnlen(pf.bdf, sizeof pf.bdf));
            if (draEnabled()) s.pfDevice = pfDeviceOf(pf, pfDeviceRead);
        }
        if (aerPortHealth) s.aerPorts = groupPorts(w.aerPortOff, w.aerPortOf, w.aerPortKey, c, g, devs, &NvidiaGpuDevice::addr);
        if (!xpuClasses[s.klass].resourceNames.empty()) {
            const kxpu_devrec &r = w.recs[c.gmem[c.goff[g]]];
            s.firstDevice = trimID(std::string((const char *)r.device_txt, std::min<size_t>(r.device_len, sizeof r.device_txt)));
        }
        iommuMap.emplace_back(std::to_string(c.gids[g]), std::move(devs));
        iommuState.push_back(std::move(s));
    }
    if (pcieTopologyAware) {
        pcieParent.assign(w.nodeParent.begin(), w.nodeParent.begin() + w.nNodes);
        pcieDepth.assign(w.nodeDepth.begin(), w.nodeDepth.begin() + w.nNodes);
    }
    buildVfVgpuDra(w);
    std::vector<kxpu_name_entry> names;
    std::vector<std::string> slotNames;  // the names classify's dev_slot indexes
    if (!c.dslot.empty()) nameTable(names, slotNames);
    for (uint32_t d = 0; d < c.nDevids; d++) {
        std::vector<std::string> groups;
        for (uint32_t k = c.doff[d]; k < c.doff[d + 1]; k++) groups.push_back(std::to_string(c.dgrp[k]));  // :169
        if (xpuClasses[c.drule[d]].vfVgpu) {  // dids[d]: the first VF carrying the entry's type key
            const kxpu_vgpukey &k = w.vkeys[c.dids[d]];
            deviceMap.emplace_back(std::string((const char *)k.key, k.len), std::move(groups));
        } else if (!c.dslot.empty() && c.dslot[d] != KXPU_NO_SLOT) {  // a configured name
            deviceMap.emplace_back(slotNames[c.dslot[d]], std::move(groups));
        } else {
            deviceMap.emplace_back(devIdString(c.dids[d]), std::move(groups));
        }
        deviceClass.push_back(c.drule[d]);
        deviceNamed.push_back(!c.dslot.empty() && c.dslot[d] != KXPU_NO_SLOT);
    }
}

// one entry per accepted function in walk order: key = PCI address, tag = its device id text packed as dev_ids packs it
std::vector<kxpu_snaprec> Plugin::snapshotOf(const PciWalk &w, const std::vector<uint64_t> *index) const {
    std::vector<kxpu_snaprec> snap;
    for (size_t i = 0; i < w.recs.size(); i++) {
        if (w.out.accept[i] == KXPU_REJECTED) continue;
        const kxpu_devrec &r = w.recs[i];
        kxpu_snaprec s;
        memset(&s, 0, sizeof s);
        memcpy(s.key, r.bdf, strnlen(r.bdf, sizeof r.bdf));
        s.iommu_group = r.iommu_group;
        s.klass = (uint32_t)recordClass(xpuClasses, r.vendor_txt, r.vendor_len, r.driver, sizeof r.driver);
        const std::string id = trimID(std::string((const char *)r.device_txt, std::min<size_t>(r.device_len, sizeof r.device_txt)));
        memcpy(&s.tag, id.data(), std::min<size_t>(id.size(), 8));
        // a vGPU VF: its type ID, so a VF whose type changed is CHANGED and gets a fresh index (a CDI name handed out for
        // the old profile never resolves to the new one); bit 63 keeps it apart from a device id text
        if (!w.vtype.empty() && xpuClasses[s.klass].vfVgpu) s.tag = 1ull << 63 | w.vtype[i];
        s.index = index ? (*index)[w.out.accept[i]] : w.out.accept[i];
        snap.push_back(s);
    }
    return snap;
}

// ---------------------------------------------------------------------------- vGPUs (mediated devices)
// canonical decimal below 2^32-1 (the domain of kxpu_mdevrec.iommu_group)
static bool parseGroup(const std::string &s, uint32_t &v) {
    if (s.empty() || s.size() > 10 || (s.size() > 1 && s[0] == '0')) return false;
    unsigned long long x = 0;
    for (char c : s) {
        if (c < '0' || c > '9') return false;
        x = x * 10 + (unsigned)(c - '0');
    }
    if (x >= 0xFFFFFFFFull) return false;
    v = (uint32_t)x;
    return true;
}

// One entry of mdevBasePath, read with the reference's read semantics through the seams: the parent's vendor
// (<uuid>/../vendor), the parent's PCI address (the basename of <uuid>/.. resolved), the `driver` and `iommu_group`
// links, and mdev_type/name.  A failed read sets its flag and ends the record, like the PCI leaf; a value outside the
// record's domain counts as that read failing (include/kxpu.h, kxpu_classify_mdev).
static void mdevRecord(Plugin &p, const std::string &name, bool isDir, kxpu_mdevrec &r) {
    memset(&r, 0, sizeof r);
    if (name.size() == sizeof r.uuid) memcpy(r.uuid, name.data(), sizeof r.uuid);  // else 36 NUL bytes: not a candidate
    if (isDir) { r.flags |= KXPU_REC_IS_DIR; return; }
    if (name.size() != sizeof r.uuid) return;
    std::string s;
    char real[PATH_MAX];
    const std::string up = p.mdevBasePath + "/" + name + "/..";
    if (!realpath(up.c_str(), real)) { r.flags |= KXPU_REC_VENDOR_ERR; return; }
    std::string parent(real);
    parent = parent.substr(parent.find_last_of('/') + 1);
    bool pok = !parent.empty() && parent.size() < sizeof r.parent;
    for (char c : parent) pok = pok && ((c >= '0' && c <= '9') || (c >= 'a' && c <= 'f') || c == ':' || c == '.');
    if (!pok) {
        fprintf(stderr, "parent of mdev %s is not a PCI address of at most 15 bytes, mdev skipped: %s\n", name.c_str(), parent.c_str());
        r.flags |= KXPU_REC_VENDOR_ERR;
        return;
    }
    memcpy(r.parent, parent.data(), parent.size());
    if (!p.readIDFromFile(p.mdevBasePath, name, "../vendor", s) || !packID(s, r.parent_vendor_txt, r.vendor_len)) {
        r.flags |= KXPU_REC_VENDOR_ERR;
        return;
    }
    if (!p.readLink(p.mdevBasePath, name, "driver", s)) { r.flags |= KXPU_REC_DRIVER_ERR; return; }
    memcpy(r.driver, s.data(), std::min<size_t>(s.size(), sizeof r.driver - 1));
    uint32_t g = 0;
    if (!p.readLink(p.mdevBasePath, name, "iommu_group", s) || !parseGroup(s, g)) { r.flags |= KXPU_REC_IOMMU_ERR; return; }
    r.iommu_group = g;
    // the parent's node; read before the name, since a record without a name can still join an existing group
    if (p.readsMdevNuma()) numaRecord([&](std::string &out) { return p.readNumaNode(p.mdevBasePath, name + "/..", out); }, r.flags, r.numa_node);
    if (!p.readIDFromFile(p.mdevBasePath, name, "mdev_type/name", s) || s.size() > sizeof r.type_name) {
        r.flags |= KXPU_REC_NAME_ERR;
        return;
    }
    memcpy(r.type_name, s.data(), s.size());
    r.name_len = (uint8_t)s.size();
}

// The entries of mdevBasePath in lexical order (filepath.Walk's order for the PCI walk).  The mdev bus directory only
// holds one level of links, so a directory inside it is recorded as such and not descended into.
Error Plugin::gatherMdevRecords(std::vector<kxpu_mdevrec> &recs, MdevWalk *w) {
    recs.clear();
    if (w) { w->parentDevice.clear(); w->pcieRoot.clear(); w->paths.clear(); w->cdevs.clear(); w->srs.clear(); }
    std::vector<int64_t> *cdevs = w && mdevCdevEnabled() ? &w->cdevs : nullptr;
    std::vector<kxpu_sriovrec> *srs = w && vgpuSriovAware ? &w->srs : nullptr;
    const bool dra = vgpuDraEnabled();
    if (!readsMdevPaths()) w = nullptr;
    DIR *d = opendir(mdevBasePath.c_str());
    if (!d) return fail("Error accessing file path \"" + mdevBasePath + "\": " + strerror(errno));
    std::vector<std::string> names;
    while (struct dirent *de = readdir(d)) {
        if (strcmp(de->d_name, ".") == 0 || strcmp(de->d_name, "..") == 0) continue;
        names.push_back(de->d_name);
    }
    closedir(d);
    std::sort(names.begin(), names.end());
    for (const std::string &n : names) {
        struct stat sb;
        const bool isDir = lstat((mdevBasePath + "/" + n).c_str(), &sb) == 0 && S_ISDIR(sb.st_mode);
        kxpu_mdevrec r;
        mdevRecord(*this, n, isDir, r);
        recs.push_back(r);
        // the vfio-dev/ read of an entry that matches an mdevCdev class (parent vendor and driver)
        if (cdevs)
            cdevs->push_back(cdevClassOf(vgpuClasses, &XpuClass::mdevCdev, r, r.parent_vendor_txt, sizeof r.parent_vendor_txt)
                                 ? readVfioCdev(mdevBasePath, n) : -1);
        if (srs) {  // the physfn link of an entry that got as far as its iommu_group link; none: the parent is no VF
            kxpu_sriovrec s;
            memset(&s, 0, sizeof s);
            std::string pf;
            if (!isDir && n.size() == sizeof r.uuid && !(r.flags & (KXPU_REC_VENDOR_ERR | KXPU_REC_DRIVER_ERR | KXPU_REC_IOMMU_ERR))) {
                mdevPhysfnReads++;
                if (readLink(mdevBasePath, n, "../physfn", pf)) {
                    if (pf.size() < sizeof s.physfn) memcpy(s.physfn, pf.data(), pf.size());
                    else s.flags |= KXPU_SR_PHYSFN_ERR;  // no PCI address is this long
                }
            }
            srs->push_back(s);
        }
        if (!w) continue;
        // the ResourceSlice and PCIe forest reads of an entry that got as far as its iommu_group link
        std::string dev, target;
        const bool grouped = !isDir && n.size() == sizeof r.uuid &&
                             !(r.flags & (KXPU_REC_VENDOR_ERR | KXPU_REC_DRIVER_ERR | KXPU_REC_IOMMU_ERR));
        if (dra && grouped && readIDFromFile(mdevBasePath, n, "../device", dev)) {
            dev = trimID(dev);
            bool ok = dev.size() <= 6;
            for (char c : dev) ok = ok && ((c >= '0' && c <= '9') || (c >= 'a' && c <= 'f'));
            if (!ok) dev.clear();
        } else {
            dev.clear();
        }
        kxpu_pcipath pp;
        memset(&pp, 0, sizeof pp);
        if (grouped && readPciPath(mdevBasePath, n, target)) pciPathRecord(target, pp);
        w->paths.push_back(pp);
        if (!dra) continue;
        w->parentDevice.push_back(dev);
        w->pcieRoot.push_back(pcieRootOf(&pp));
    }
    return Error();
}

Error Plugin::checkVgpuClasses() const {
    std::vector<const XpuClass *> all;
    for (const XpuClass &c : xpuClasses) all.push_back(&c);
    for (const XpuClass &c : vgpuClasses) all.push_back(&c);
    for (size_t v = xpuClasses.size(); v < all.size(); v++)
        for (size_t o = 0; o < all.size(); o++)
            if (o != v && (all[o]->cdiKind == all[v]->cdiKind || all[o]->cdiFileStem == all[v]->cdiFileStem))
                return fail("vGPU class " + all[v]->vendor + "/" + all[v]->driver + ": CDI kind and file stem must differ from every other class's");
    if (vgpuClasses.size() > KXPU_MAX_RULES) return fail("more vGPU classes than KXPU_MAX_RULES");
    for (const XpuClass &c : vgpuClasses)
        if (c.vfioCdev) return fail("vGPU class " + c.vendor + "/" + c.driver + " (" + c.cdiKind + "): vfioCdev applies to passthrough classes only; a vGPU class sets mdevCdev");
    return checkPassthroughClasses(xpuClasses);
}

// the parse call of the mdev resume: kxpu_cdi_parse_mdev into the record type of the vGPU spec paths (cdiRecord)
static int32_t parseMdevGroup(kxpu_ctx *ctx, int32_t fmt, const char *kind, const uint8_t *doc, size_t len, kxpu_mdevcdev *out,
                              size_t cap, size_t *n) {
    std::vector<kxpu_mdevcdi> d(cap);
    const int32_t rc = kxpu_cdi_parse_mdev(ctx, fmt, kind, doc, len, d.data(), cap, n);
    if (rc == KXPU_OK)
        for (size_t i = 0; i < *n; i++) {
            memset(&out[i], 0, sizeof out[i]);
            out[i].dev = d[i];
        }
    return rc;
}

Error Plugin::createMdevMap() {
    mdevMap.clear();
    typeMap.clear();
    mdevState.clear();
    typeClass.clear();
    mdev_.snap.clear();
    mdev_.next = 0;
    if (vgpuClasses.empty()) return Error();  // nothing under mdevBasePath is read
    Error e = checkVgpuClasses();
    if (e) return e;
    mdev_.haveGen = mdevGeneration && mdevGeneration(mdev_.gen);
    MdevWalk w;
    e = firstWalk(w, mdev_);
    if (e || !resumeIndices) return e;
    const uint64_t stateNext = resume_.stateRead ? resume_.stateMdev : 0;
    std::vector<kxpu_snaprec> prev;
    uint64_t next = 0;
    previousEntries<kxpu_mdevcdev>(vgpuClasses, parseMdevGroup, stateNext, resume_.mdev, prev, next);
    return resume(w, mdev_, resume_.mdev, stateNext, std::move(prev), next);
}

Error Plugin::classify(MdevWalk &w) {
    Error e = gatherMdevRecords(w.recs, &w);
    if (e) { fprintf(stderr, "%s\n", e.message.c_str()); }  // like the PCI walk: an unreadable bus is an empty one
    const std::vector<kxpu_mdevrec> &recs = w.recs;
    const size_t n = recs.size();
    if (vgpuSriovAware) {  // each mdev's PF in the PCI walk, which ran first
        w.pfOf.assign(n + 1, KXPU_NO_PF);
        const int32_t rc = kxpu_mdev_pf(ctx_, pciRecs_.data(), pciRecs_.size(), recs.data(), w.srs.data(), n, w.pfOf.data());
        if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_mdev_pf", rc);
    }
    ClassifyResult &c = w.out;
    kxpu_classify_out out = c.wire(n);
    const std::vector<kxpu_xpu_rule> rules = classRules(vgpuClasses);
    const bool topo = readsMdevNuma();
    int32_t rc = topo ? kxpu_classify_mdev_topo(ctx_, rules.data(), rules.size(), recs.data(), n, &out, c.drule.data(), c.gnuma.data())
                      : kxpu_classify_mdev(ctx_, rules.data(), rules.size(), recs.data(), n, &out, c.drule.data());
    if (rc != KXPU_OK) return kxfail(ctx_, topo ? "kxpu_classify_mdev_topo" : "kxpu_classify_mdev", rc);
    c.nGroups = out.n_groups;
    c.nDevids = out.n_devids;
    std::vector<uint32_t> first(out.n_devids);
    for (uint32_t d = 0; d < out.n_devids; d++) first[d] = (uint32_t)c.dids[d];
    w.koff.assign(first.size() + 1, 0);
    size_t need = 0;
    rc = kxpu_mdev_names(ctx_, recs.data(), n, first.data(), first.size(), nullptr, 0, w.koff.data(), &need);
    if (rc != KXPU_OK && rc != KXPU_E_NOSPACE) return kxfail(ctx_, "kxpu_mdev_names", rc);
    w.keys.assign(need ? need : 1, 0);
    rc = kxpu_mdev_names(ctx_, recs.data(), n, first.data(), first.size(), w.keys.data(), need, w.koff.data(), &need);
    if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_mdev_names", rc);
    if (vgpuPcieTopologyAware) {  // the forest of the walk, one node per group, every mdev below its parent function
        const size_t cap = (size_t)KXPU_PCIE_MAX_DEPTH * c.nGroups + 1;
        w.gnode.assign(c.nGroups + 1, KXPU_PCIE_NO_NODE);
        w.nodeKey.assign(cap, 0); w.nodeParent.assign(cap, 0); w.nodeDepth.assign(cap, 0);
        rc = kxpu_pcie_tree_mdev(ctx_, recs.data(), w.paths.data(), n, c.goff.data(), c.gmem.data(), c.nGroups, w.gnode.data(),
                                 w.nodeKey.data(), w.nodeParent.data(), w.nodeDepth.data(), &w.nNodes);
        if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_pcie_tree_mdev", rc);
    }
    if (draVgpuPcie && vgpuDraEnabled()) {  // each group's root port and switch, from the links the DRA walk reads
        w.rootPort.assign(c.nGroups + 1, KXPU_PCIE_NO_KEY);
        w.pcieSwitch.assign(c.nGroups + 1, KXPU_PCIE_NO_KEY);
        rc = kxpu_pcie_ports_mdev(ctx_, recs.data(), w.paths.data(), n, c.goff.data(), c.gmem.data(), c.nGroups,
                                  w.rootPort.data(), w.pcieSwitch.data());
        if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_pcie_ports_mdev", rc);
    }
    if (aerPortHealth) {  // the ports above every mdev's parent, from the links read above
        w.aerPortOff.assign(n + 1, 0);
        w.aerPortOf.assign((size_t)KXPU_PCIE_MAX_DEPTH * n + 1, 0);
        w.aerPortKey.assign((size_t)KXPU_PCIE_MAX_DEPTH * n + 1, 0);
        uint32_t nk = 0;
        rc = kxpu_aer_ports_mdev(ctx_, recs.data(), w.paths.data(), n, w.aerPortOff.data(), w.aerPortOf.data(),
                                 w.aerPortKey.data(), &nk);
        if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_aer_ports_mdev", rc);
        w.aerPortOf.resize(w.aerPortOff[n]);
        w.aerPortKey.resize(nk);
    }
    return Error();
}

void Plugin::buildMaps(const MdevWalk &w, const std::vector<uint64_t> *index) {
    mdevMap.clear();
    typeMap.clear();
    mdevState.clear();
    typeClass.clear();
    const ClassifyResult &c = w.out;
    std::map<uint32_t, size_t> groupClass = groupClasses(c);
    for (uint32_t g = 0; g < c.nGroups; g++) {
        std::vector<MdevDevice> devs;
        for (uint32_t k = c.goff[g]; k < c.goff[g + 1]; k++) {
            const kxpu_mdevrec &r = w.recs[c.gmem[k]];
            const uint64_t idx = index ? (*index)[c.accept[c.gmem[k]]] : c.accept[c.gmem[k]];
            MdevDevice m{std::string(r.uuid, sizeof r.uuid), std::string(r.parent, strnlen(r.parent, sizeof r.parent)), idx, 0};
            m.vgpuClass = recordClass(vgpuClasses, r.parent_vendor_txt, r.vendor_len, r.driver, sizeof r.driver);
            if (!w.cdevs.empty()) m.cdev = w.cdevs[c.gmem[k]];
            devs.push_back(std::move(m));
        }
        GroupState<kxpu_dramdev> s;
        s.klass = groupClass[c.gids[g]];
        if (topologyAware) s.numa = c.gnuma[g];
        if (vgpuPcieTopologyAware) s.pcieNode = w.gnode[g];
        if (!w.rootPort.empty()) { s.rootPort = w.rootPort[g]; s.pcieSwitch = w.pcieSwitch[g]; }
        if (vgpuSriovAware && w.pfOf[c.gmem[c.goff[g]]] != KXPU_NO_PF) {
            const kxpu_devrec &pf = pciRecs_[w.pfOf[c.gmem[c.goff[g]]]];
            s.pf.assign(pf.bdf, strnlen(pf.bdf, sizeof pf.bdf));
        }
        if (aerPortHealth) s.aerPorts = groupPorts(w.aerPortOff, w.aerPortOf, w.aerPortKey, c, g, devs, &MdevDevice::parent);
        if (vgpuClasses[s.klass].mdevCdev)  // an mdev without a cdev: VFIO cannot open it
            for (const MdevDevice &m : devs)
                if (m.cdev < 0) { s.blocker = m.uuid + " has no VFIO cdev"; s.blockerKind = KXPU_MR_VFIO_CDEV_MISSING; break; }
        mdevMap.emplace_back(std::to_string(c.gids[g]), std::move(devs));
        mdevState.push_back(std::move(s));
    }
    for (uint32_t d = 0; d < c.nDevids; d++) {
        std::vector<std::string> groups;
        for (uint32_t k = c.doff[d]; k < c.doff[d + 1]; k++) groups.push_back(std::to_string(c.dgrp[k]));
        typeMap.emplace_back(std::string((const char *)w.keys.data() + w.koff[d], w.koff[d + 1] - w.koff[d]), std::move(groups));
        typeClass.push_back(c.drule[d]);
    }
    if (vgpuPcieTopologyAware) {
        mdevPcieParent.assign(w.nodeParent.begin(), w.nodeParent.begin() + w.nNodes);
        mdevPcieDepth.assign(w.nodeDepth.begin(), w.nodeDepth.begin() + w.nNodes);
    }
    buildMdevDra(w);
}

// the dra record of every mdevState entry (vgpuDraEnabled only): one kxpu_dramdev per group from its first mdev; the
// parents' model names come from one getDeviceNames call over the distinct (vendor, device) ids
void Plugin::buildMdevDra(const MdevWalk &w) {
    if (!vgpuDraEnabled()) return;
    const ClassifyResult &c = w.out;
    std::map<uint32_t, std::string> keyOf;  // group id -> type key of its device-map entry
    for (uint32_t d = 0; d < c.nDevids; d++)
        for (uint32_t k = c.doff[d]; k < c.doff[d + 1]; k++)
            keyOf[c.dgrp[k]] = std::string((const char *)w.keys.data() + w.koff[d], w.koff[d + 1] - w.koff[d]);
    std::map<std::pair<std::string, std::string>, size_t> idAt;  // (vendor, device) -> position in the lookup batch
    std::vector<std::string> ids, vendors;
    std::vector<std::pair<std::string, std::string>> idOf;  // per group
    std::vector<std::pair<uint32_t, std::pair<std::string, std::string>>> pfIds;  // (group, its PF's ids)
    std::map<std::string, std::string> pfDeviceRead;  // PF address -> its device file, for PFs the walk did not read
    for (uint32_t g = 0; g < c.nGroups; g++) {
        const uint32_t first = c.gmem[c.goff[g]];
        const kxpu_mdevrec &r = w.recs[first];
        kxpu_dramdev d;
        memset(&d, 0, sizeof d);
        const std::string key = keyOf[c.gids[g]];
        memcpy(d.mdev_type, key.data(), std::min(key.size(), sizeof d.mdev_type));
        memcpy(d.uuid, r.uuid, sizeof d.uuid);
        d.iommu_group = r.iommu_group;
        memcpy(d.parent, r.parent, strnlen(r.parent, sizeof r.parent));
        const std::string vendor = trimID(std::string((const char *)r.parent_vendor_txt, std::min<size_t>(r.vendor_len, sizeof r.parent_vendor_txt)));
        memcpy(d.vendor, vendor.data(), std::min(vendor.size(), sizeof d.vendor));
        const std::string device = first < w.parentDevice.size() ? w.parentDevice[first] : std::string();
        memcpy(d.device, device.data(), std::min(device.size(), sizeof d.device));
        const std::string root = first < w.pcieRoot.size() ? w.pcieRoot[first] : std::string();
        memcpy(d.pcie_root, root.data(), std::min(root.size(), sizeof d.pcie_root));
        d.numa_mask = c.gnuma.size() > g ? c.gnuma[g] : 0;
        mdevState[g].dra = d;
        idOf.emplace_back(vendor, device);
        if (!device.empty() && idAt.emplace(idOf.back(), ids.size()).second) {
            ids.push_back(device);
            vendors.push_back(vendor);
        }
        if (!mdevState[g].pf.empty()) {  // vgpuSriovAware: the PF's ids from its own record in the PCI walk
            const kxpu_devrec &pf = pciRecs_[w.pfOf[first]];
            const std::string pv = trimID(std::string((const char *)pf.vendor_txt, std::min<size_t>(pf.vendor_len, sizeof pf.vendor_txt)));
            std::string pd = (pf.flags & KXPU_REC_DEVICE_ERR) ? std::string()
                             : trimID(std::string((const char *)pf.device_txt, std::min<size_t>(pf.device_len, sizeof pf.device_txt)));
            if (pd.empty() && !pfDeviceRead.count(mdevState[g].pf)) {  // a PF that is no class candidate: the walk left
                std::string raw;                                       // its device id unread; read it once here
                pfDeviceRead[mdevState[g].pf] = readIDFromFile(basePath, mdevState[g].pf, "device", raw) ? trimID(raw) : "";
            }
            if (pd.empty()) pd = pfDeviceRead[mdevState[g].pf];
            bool ok = pd.size() <= 6;
            for (char ch : pd) ok = ok && ((ch >= '0' && ch <= '9') || (ch >= 'a' && ch <= 'f'));
            if (!ok) pd.clear();
            mdevState[g].pfDevice = pd;
            if (!pd.empty() && idAt.emplace(std::make_pair(pv, pd), ids.size()).second) {
                ids.push_back(pd);
                vendors.push_back(pv);
            }
            pfIds.emplace_back(g, std::make_pair(pv, pd));
        }
    }
    const std::vector<std::string> names = ids.empty() ? std::vector<std::string>() : getDeviceNames(ids, vendors);
    for (const auto &gi : pfIds) {
        if (gi.second.second.empty()) continue;
        const std::string &name = names[idAt[gi.second]];
        mdevState[gi.first].pfProduct = (name.empty() ? gi.second.second : name).substr(0, sizeof(kxpu_dramdev::product));
    }
    for (size_t g = 0; g < mdevState.size(); g++) {
        if (idOf[g].second.empty()) continue;  // no device id: no productName
        const std::string &name = names[idAt[idOf[g]]];
        const std::string &product = name.empty() ? idOf[g].second : name;
        kxpu_dramdev &d = *mdevState[g].dra;
        d.product_len = (uint8_t)std::min(product.size(), sizeof d.product);
        memcpy(d.product, product.data(), d.product_len);
    }
}

// the VF-vGPU record of every iommuState entry of a class with a vgpuDraDriver (vfVgpuDraEnabled only) whose first
// member is a VF with a named type: one kxpu_dravfvgpu from that VF and its PF.  The PF's vendor and device ids come from
// its own record in this walk; the PFs' model names from one getDeviceNames call over the distinct (vendor, device) ids
void Plugin::buildVfVgpuDra(const PciWalk &w) {
    if (!vfVgpuDraEnabled()) return;
    const ClassifyResult &c = w.out;
    std::map<std::string, size_t> recAt;  // PCI address -> record
    for (size_t i = 0; i < w.recs.size(); i++) recAt.emplace(std::string(w.recs[i].bdf, strnlen(w.recs[i].bdf, sizeof w.recs[i].bdf)), i);
    std::map<std::pair<std::string, std::string>, size_t> idAt;  // (vendor, device) -> position in the lookup batch
    std::vector<std::string> ids, vendors;
    std::vector<std::pair<size_t, std::pair<std::string, std::string>>> idOf;  // (group, its PF's ids)
    auto idText = [](const uint8_t *txt, uint8_t len, size_t cap) {
        return trimID(std::string((const char *)txt, std::min<size_t>(len, cap)));
    };
    for (uint32_t g = 0; g < c.nGroups; g++) {
        const uint32_t first = c.gmem[c.goff[g]];
        const kxpu_devrec &r = w.recs[first];
        const XpuClass &k = xpuClasses[iommuState[g].klass];
        if (k.vgpuDraDriver.empty() || !xpuClasses[recordClass(xpuClasses, r.vendor_txt, r.vendor_len, r.driver, sizeof r.driver)].vfVgpu ||
            w.vstatus[first] != KXPU_VT_NAMED || w.physfn[first].empty())
            continue;
        kxpu_dravfvgpu d;
        memset(&d, 0, sizeof d);
        memcpy(d.type_key, w.vkeys[first].key, std::min<size_t>(w.vkeys[first].len, sizeof d.type_key));
        d.type_id = w.vtype[first];
        memcpy(d.bdf, r.bdf, strnlen(r.bdf, sizeof r.bdf));
        const std::string &pf = w.physfn[first];
        memcpy(d.parent, pf.data(), std::min(pf.size(), sizeof d.parent));
        const std::string root = pcieRootOf(w.paths.size() > first ? &w.paths[first] : nullptr);
        memcpy(d.pcie_root, root.data(), root.size());
        std::string vendor = idText(r.vendor_txt, r.vendor_len, sizeof r.vendor_txt), device;
        auto at = recAt.find(pf);
        if (at != recAt.end()) {
            const kxpu_devrec &p = w.recs[at->second];
            if (!(p.flags & KXPU_REC_VENDOR_ERR)) vendor = idText(p.vendor_txt, p.vendor_len, sizeof p.vendor_txt);
            if (p.device_len && !(p.flags & KXPU_REC_DEVICE_ERR)) device = idText(p.device_txt, p.device_len, sizeof p.device_txt);
        }
        memcpy(d.vendor, vendor.data(), std::min(vendor.size(), sizeof d.vendor));
        memcpy(d.device, device.data(), std::min(device.size(), sizeof d.device));
        d.numa_mask = c.gnuma.size() > g ? c.gnuma[g] : 0;
        d.iommu_group = r.iommu_group;
        iommuState[g].vfVgpuDra = d;
        idOf.emplace_back(g, std::make_pair(vendor, device));
        if (!device.empty() && idAt.emplace(idOf.back().second, ids.size()).second) {
            ids.push_back(device);
            vendors.push_back(vendor);
        }
    }
    const std::vector<std::string> names = ids.empty() ? std::vector<std::string>() : getDeviceNames(ids, vendors);
    for (const auto &gi : idOf) {
        if (gi.second.second.empty()) continue;  // no device id: no productName
        const std::string &name = names[idAt[gi.second]];
        const std::string &product = name.empty() ? gi.second.second : name;
        kxpu_dravfvgpu &d = *iommuState[gi.first].vfVgpuDra;
        d.product_len = (uint8_t)std::min(product.size(), sizeof d.product);
        memcpy(d.product, product.data(), d.product_len);
    }
}

static uint64_t fnv1a64(const std::string &s) {
    uint64_t h = 0xCBF29CE484222325ull;
    for (unsigned char c : s) h = (h ^ c) * 0x100000001B3ull;
    return h;
}

// one entry per accepted mdev in walk order: key = UUID, tag = FNV-1a 64 of the type key of the resource its group is
// served under (the type key of the group's device-map entry: known on the host without another GPU call)
std::vector<kxpu_snaprec> Plugin::snapshotOf(const MdevWalk &w, const std::vector<uint64_t> *index) const {
    const ClassifyResult &c = w.out;
    std::map<uint32_t, uint64_t> groupTag;
    for (uint32_t d = 0; d < c.nDevids; d++) {
        const uint64_t t = fnv1a64(std::string((const char *)w.keys.data() + w.koff[d], w.koff[d + 1] - w.koff[d]));
        for (uint32_t k = c.doff[d]; k < c.doff[d + 1]; k++) groupTag[c.dgrp[k]] = t;
    }
    std::vector<kxpu_snaprec> snap;
    for (size_t i = 0; i < w.recs.size(); i++) {
        if (c.accept[i] == KXPU_REJECTED) continue;
        const kxpu_mdevrec &r = w.recs[i];
        kxpu_snaprec s;
        memset(&s, 0, sizeof s);
        memcpy(s.key, r.uuid, sizeof r.uuid);
        s.iommu_group = r.iommu_group;
        s.klass = (uint32_t)recordClass(vgpuClasses, r.parent_vendor_txt, r.vendor_len, r.driver, sizeof r.driver);
        s.tag = groupTag[r.iommu_group];
        s.index = index ? (*index)[c.accept[i]] : c.accept[i];
        snap.push_back(s);
    }
    return snap;
}

// group id -> position in a walk's map, which is also its position in the walk's states
template <typename V>
static std::map<std::string, size_t> positions(const OrderedMap<V> &m) {
    std::map<std::string, size_t> at;
    for (size_t g = 0; g < m.size(); g++) at.emplace(m[g].first, g);
    return at;
}

// the state of group `id` of a walk (its map and states, same positions); nullptr when the walk has no such group
template <typename V, typename Dra>
static const GroupState<Dra> *stateOf(const OrderedMap<V> &m, const std::vector<GroupState<Dra>> &state, const std::string &id) {
    for (size_t g = 0; g < m.size(); g++)
        if (m[g].first == id) return &state[g];
    return nullptr;
}

// The pci.ids file into page-locked memory the GPU can address (kxpu_pinned_alloc): with text, keys and rows in
// such buffers kxpu_pciids_join copies nothing -- one cooperative kernel pulls the text over PCIe, builds the
// table and writes the row handles back (include/kxpu.h).  Falls back to ordinary memory when pinning fails.
namespace {
struct PinnedBuf {
    kxpu_ctx *ctx;
    void *p = nullptr;
    bool pinned = false;
    size_t n = 0;
    PinnedBuf(kxpu_ctx *c, size_t bytes) : ctx(c), n(bytes) {
        if (kxpu_pinned_alloc(ctx, bytes ? bytes : 16, &p) == KXPU_OK && p) pinned = true;
        else p = malloc(bytes ? bytes : 16);
    }
    ~PinnedBuf() {
        if (pinned) kxpu_pinned_free(ctx, p);
        else free(p);
    }
    PinnedBuf(const PinnedBuf &) = delete;
    PinnedBuf &operator=(const PinnedBuf &) = delete;
};
}  // namespace

// First use: ONE kxpu_pciids_join call reads the file (device_plugin.go:210), builds the table and joins `keys`
// (the start-up batch of createDevicePlugins, device_plugin.go:91-105).  keys may be empty (load only).
Error Plugin::loadAndJoin(const std::vector<uint32_t> &keys, std::vector<int32_t> &rows) {
    FILE *f = fopen(pciIdsFilePath.c_str(), "rb");  // device_plugin.go:210
    if (!f) return fail("Error opening pci ids file " + pciIdsFilePath);
    std::vector<uint8_t> head;
    size_t n = 0;
    if (fseek(f, 0, SEEK_END) == 0) {
        const long sz = ftell(f);
        if (sz > 0) n = (size_t)sz;
        rewind(f);
    }
    PinnedBuf text(ctx_, n), hk(ctx_, keys.size() * 4), hr(ctx_, keys.size() * 4);
    if (!text.p || !hk.p || !hr.p) { fclose(f); return fail("out of memory reading " + pciIdsFilePath); }
    const size_t got = n ? fread(text.p, 1, n, f) : 0;
    fclose(f);
    if (!keys.empty()) memcpy(hk.p, keys.data(), keys.size() * 4);
    const int32_t rc = kxpu_pciids_join(ctx_, (const uint8_t *)text.p, got, (const uint32_t *)hk.p, keys.size(), (int32_t *)hr.p, &table_);
    if (rc != KXPU_OK) { table_ = nullptr; return kxfail(ctx_, "kxpu_pciids_join", rc); }
    rows.assign((const int32_t *)hr.p, (const int32_t *)hr.p + keys.size());
    return Error();
}

Error Plugin::ensureTable() {
    if (table_) return Error();
    std::vector<int32_t> none;
    return loadAndJoin({}, none);
}

static bool parseHex4(const std::string &s, uint32_t &v) {
    if (s.size() != 4) return false;
    v = 0;
    for (char c : s) {
        uint32_t d;
        if (c >= '0' && c <= '9') d = (uint32_t)(c - '0');
        else if (c >= 'a' && c <= 'f') d = (uint32_t)(c - 'a' + 10);
        else return false;
        v = v * 16 + d;
    }
    return true;
}

// getDeviceName, device_plugin.go:208-259, for a whole batch of device ids: ONE join and ONE name
// gather through the ABI (cgo calls stay coarse, SURVEY H7).  "" means "not found" exactly like the
// reference; sysfs ids are four lowercase hex digits, anything else is treated as not found.
// The key of id i is (vendors[i] << 16) | id; a vendor that is not four lowercase hex digits
// never names anything, so that device falls back to its raw id like a miss (:100-103).
std::vector<std::string> Plugin::getDeviceNames(const std::vector<std::string> &deviceIDs, const std::vector<std::string> &vendors) {
    std::vector<std::string> out(deviceIDs.size());
    std::vector<uint32_t> keys;
    std::vector<size_t> where;
    for (size_t i = 0; i < deviceIDs.size(); i++) {
        uint32_t d, v;
        if (parseHex4(vendors[i], v) && parseHex4(deviceIDs[i], d)) { keys.push_back((v << 16) | d); where.push_back(i); }
    }
    std::vector<int32_t> rows(keys.size(), KXPU_ROW_MISS);
    if (!table_) {
        // start-up: file -> table -> row handles of the whole batch in one call
        Error e = loadAndJoin(keys, rows);
        if (e) { fprintf(stderr, "%s\n", e.message.c_str()); return out; }  // :211-214
        if (keys.empty()) return out;
    } else {
        if (keys.empty()) return out;
        if (kxpu_lookup(ctx_, table_, keys.data(), keys.size(), rows.data()) != KXPU_OK) return out;
    }
    std::vector<uint32_t> offs(keys.size() + 1);
    size_t need = 0;
    int32_t rc = kxpu_names(ctx_, table_, rows.data(), rows.size(), nullptr, 0, offs.data(), &need);
    if (rc != KXPU_OK && rc != KXPU_E_NOSPACE) return out;
    std::vector<uint8_t> blob(need ? need : 1);
    if (need && kxpu_names(ctx_, table_, rows.data(), rows.size(), blob.data(), need, offs.data(), &need) != KXPU_OK) return out;
    for (size_t k = 0; k < keys.size(); k++) {
        if (rows[k] == KXPU_ROW_MISS) {
            const std::string &vendor = vendors[where[k]], &id = deviceIDs[where[k]];
            if (vendor == "10de") fprintf(stderr, "Could not find NVIDIA device with id: %s\n", id.c_str());  // :234
            else fprintf(stderr, "Could not find device %s:%s\n", vendor.c_str(), id.c_str());
            continue;
        }
        out[where[k]].assign((const char *)blob.data() + offs[k], offs[k + 1] - offs[k]);
    }
    return out;
}

std::string Plugin::getDeviceName(const std::string &deviceID) { return getDeviceNames({deviceID}, {defaultXpuClass().vendor})[0]; }

static Error writeSpecFile(const std::string &file_path, const std::vector<uint8_t> &doc, size_t len, bool &written) {
    written = false;
    FILE *f = fopen(file_path.c_str(), "wb");  // os.Create
    if (!f) {
        printf("Error creating file: %s\n", strerror(errno));  // spec.go:95: printed and swallowed
        return Error();
    }
    size_t w = fwrite(doc.data(), 1, len, f);
    fclose(f);
    if (w != len) { printf("Error writing to file\n"); return Error(); }
    written = true;
    printf("Data successfully written to file\n");  // spec.go:126
    return Error();
}

// The rediscovery writer: nothing when the file already holds these bytes; else <dir>/.<name>.tmp, fsync, rename, so
// that a reader sees the old document or the new one, never a partial one (a reader that opened the old file keeps
// reading the old bytes).  The CDI cache only loads *.json / *.yaml, so it ignores the .tmp file.
static Error writeSpecFileAtomic(const std::string &file_path, const uint8_t *doc, size_t len, bool &written) {
    written = false;
    if (FILE *f = fopen(file_path.c_str(), "rb")) {
        std::vector<uint8_t> old(len + 1);
        const size_t got = fread(old.data(), 1, len + 1, f);
        fclose(f);
        if (got == len && memcmp(old.data(), doc, len) == 0) return Error();
    }
    const size_t slash = file_path.find_last_of('/');
    const std::string dir = slash == std::string::npos ? std::string(".") : file_path.substr(0, slash);
    const std::string name = slash == std::string::npos ? file_path : file_path.substr(slash + 1);
    const std::string tmp = dir + "/." + name + ".tmp";
    int fd = open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    if (fd < 0) return fail("Error creating file " + tmp + ": " + strerror(errno));
    size_t off = 0;
    while (off < len) {
        ssize_t k = write(fd, doc + off, len - off);
        if (k < 0 && errno == EINTR) continue;
        if (k <= 0) break;
        off += (size_t)k;
    }
    const bool ok = off == len && fsync(fd) == 0;
    close(fd);
    if (!ok || rename(tmp.c_str(), file_path.c_str()) != 0) {
        const std::string err = strerror(errno);
        unlink(tmp.c_str());
        return fail("Error writing file " + file_path + ": " + err);
    }
    written = true;
    return Error();
}

Error writeSpecFileAtomicForTests(const std::string &file_path, const uint8_t *doc, size_t len, bool &written) {
    return writeSpecFileAtomic(file_path, doc, len, written);
}

Error Plugin::writeSpec(const std::string &path, const std::vector<uint8_t> &doc, size_t len, bool &written) {
    if (!atomicSpecs_) return writeSpecFile(path, doc, len, written);  // start-up: the reference's os.Create path
    Error e = writeSpecFileAtomic(path, doc.data(), len, written);
    if (written) specsWritten_.push_back(path);
    return e;
}

// the CDI record of one device of group `group`: the passthrough spec paths hold one record type for every layout, the
// untyped layouts read each record's dev
static kxpu_vfvgpucdi cdiRecord(const std::string &group, const NvidiaGpuDevice &dev) {
    kxpu_vfvgpucdi d;
    memset(&d, 0, sizeof d);
    strncpy(d.dev.bdf, dev.addr.c_str(), sizeof d.dev.bdf - 1);
    d.dev.iommu_group = (uint32_t)strtoul(group.c_str(), nullptr, 10);
    d.dev.vfio_cdev = dev.cdev < 0 ? 0u : (uint32_t)dev.cdev;
    d.dev.index = dev.index;
    d.type_id = dev.vgpuType;
    d.key_len = (uint8_t)std::min(dev.vgpuKey.size(), sizeof d.key);
    memcpy(d.key, dev.vgpuKey.data(), d.key_len);
    return d;
}
static bool hasCdev(const NvidiaGpuDevice &dev) { return dev.cdev >= 0; }
static bool hasCdev(const MdevDevice &m) { return m.cdev >= 0; }
// the vGPU spec paths hold one record type for both node layouts: the group layout reads and writes each record's dev
static kxpu_mdevcdev cdiRecord(const std::string &group, const MdevDevice &m) {
    kxpu_mdevcdev d;
    memset(&d, 0, sizeof d);
    memcpy(d.dev.uuid, m.uuid.data(), std::min(m.uuid.size(), sizeof d.dev.uuid));
    strncpy(d.dev.parent, m.parent.c_str(), sizeof d.dev.parent - 1);
    d.dev.iommu_group = (uint32_t)strtoul(group.c_str(), nullptr, 10);
    d.dev.index = m.index;
    d.vfio_cdev = m.cdev < 0 ? 0u : (uint32_t)m.cdev;
    return d;
}
static const kxpu_cdidev &cdiBase(const kxpu_vfvgpucdi &r) { return r.dev; }
static const kxpu_mdevcdi &cdiBase(const kxpu_mdevcdev &r) { return r.dev; }
template <int32_t (*emit)(kxpu_ctx *, int32_t, const char *, const kxpu_cdidev *, size_t, uint8_t *, size_t, size_t *)>
static int32_t emitUntyped(kxpu_ctx *ctx, int32_t fmt, const char *kind, const kxpu_vfvgpucdi *devs, size_t n, uint8_t *out,
                           size_t cap, size_t *len) {
    std::vector<kxpu_cdidev> d(n);
    for (size_t i = 0; i < n; i++) d[i] = devs[i].dev;
    return emit(ctx, fmt, kind, d.data(), n, out, cap, len);
}
static int32_t emitMdevGroup(kxpu_ctx *ctx, int32_t fmt, const char *kind, const kxpu_mdevcdev *devs, size_t n, uint8_t *out,
                             size_t cap, size_t *len) {
    std::vector<kxpu_mdevcdi> d(n);
    for (size_t i = 0; i < n; i++) d[i] = devs[i].dev;
    return kxpu_cdi_emit_mdev(ctx, fmt, kind, d.data(), n, out, cap, len);
}

// One file per class, <stem>.yaml|.json, with that class's kind and only the devices of its entries in ascending index
// (Go ranges over the map in random order, device_plugin.go:59); a class without devices gets the empty document (the
// reference writes one for zero devices too).  The files written go to `files`.
template <typename Dev, typename Rec>
Error Plugin::generateClassSpecs(const std::vector<XpuClass> &classes, const OrderedMap<std::vector<Dev>> &m,
                                 const std::vector<size_t> &entryClass, int32_t fmt, const char *what,
                                 int32_t (*emit)(kxpu_ctx *, int32_t, const char *, const Rec *, size_t, uint8_t *, size_t, size_t *),
                                 std::vector<std::string> &files) {
    std::vector<std::vector<Rec>> per(classes.size());
    for (size_t g = 0; g < m.size(); g++) {
        bool cdevs = true;  // a vfioCdev / mdevCdev class's spec leaves out a group with a member without a cdev
        for (const Dev &dev : m[g].second) cdevs &= hasCdev(dev);
        if ((classes[entryClass[g]].vfioCdev || classes[entryClass[g]].mdevCdev) && !cdevs) continue;
        for (const Dev &dev : m[g].second) per[entryClass[g]].push_back(cdiRecord(m[g].first, dev));
    }
    for (size_t c = 0; c < classes.size(); c++) {
        std::vector<Rec> &devs = per[c];
        std::sort(devs.begin(), devs.end(), [](const Rec &a, const Rec &b) { return cdiBase(a).index < cdiBase(b).index; });
        const char *kind = classes[c].cdiKind.c_str();
        size_t len = 0;
        auto *fn = emit;
        if constexpr (std::is_same<Rec, kxpu_vfvgpucdi>::value) {
            if (classes[c].vfioCdev) fn = emitUntyped<kxpu_cdi_emit_cdev>;
            // resumeIndices: a vfVgpu class's spec carries each VF's type, which a restart reads back
            if (classes[c].vfVgpu && resumeIndices) fn = classes[c].vfioCdev ? kxpu_cdi_emit_vf_vgpu_cdev : kxpu_cdi_emit_vf_vgpu;
        }
        if constexpr (std::is_same<Rec, kxpu_mdevcdev>::value)
            if (classes[c].mdevCdev) fn = kxpu_cdi_emit_mdev_cdev;
        int32_t rc = fn(ctx_, fmt, kind, devs.data(), devs.size(), nullptr, 0, &len);
        if (rc != KXPU_OK && rc != KXPU_E_NOSPACE) return kxfail(ctx_, what, rc);
        std::vector<uint8_t> doc(len ? len : 1);
        rc = fn(ctx_, fmt, kind, devs.data(), devs.size(), doc.data(), len, &len);
        if (rc != KXPU_OK) return kxfail(ctx_, what, rc);
        const std::string file_path = cdiConfigPath + classes[c].cdiFileStem + (fmt == KXPU_FMT_YAML ? ".yaml" : ".json");  // spec.go:92
        bool written = false;
        Error e = writeSpec(file_path, doc, len, written);  // os.Create at start-up (spec.go:93-126)
        if (e) return e;
        if (written || atomicSpecs_) files.push_back(file_path);
    }
    return Error();
}

// generateCDISpec, device_plugin.go:55-80 + CdiSpec.Save, cdi/spec.go:85-127, one file per class
Error Plugin::generateCDISpec(const OrderedMap<std::vector<NvidiaGpuDevice>> &m, const std::string &format) {
    cdiFiles.clear();
    std::map<std::string, size_t> classOf;  // group -> class, from the maps of the last walk
    // sriovAware: a group with an SR-IOV reason, which VFIO would refuse to open; resetCheck: one VFIO cannot reset
    std::set<std::string> withheld;
    for (size_t g = 0; g < iommuMap.size(); g++) {
        classOf.emplace(iommuMap[g].first, iommuState[g].klass);
        if (!iommuState[g].sriov.empty() || !iommuState[g].reset.empty()) withheld.insert(iommuMap[g].first);
    }
    OrderedMap<std::vector<NvidiaGpuDevice>> served;  // m without them (only built when some group is withheld)
    std::vector<size_t> entryClass;
    for (const auto &kv : m) {
        if (withheld.count(kv.first)) continue;
        if (!withheld.empty()) served.push_back(kv);
        auto it = classOf.find(kv.first);
        entryClass.push_back(it == classOf.end() ? 0 : it->second);
    }
    const int32_t fmt = format == "YAML" ? KXPU_FMT_YAML : KXPU_FMT_JSON;  // spec.go:86-89,102-114
    Error e = generateClassSpecs(xpuClasses, withheld.empty() ? m : served, entryClass, fmt, "kxpu_cdi_emit_kind",
                                 emitUntyped<kxpu_cdi_emit_kind>, cdiFiles);
    if (!cdiFiles.empty()) lastCdiFile = cdiFiles.back();
    return e;
}

// One CDI spec per vGPU class: the mdevs of the class's groups in ascending index; a class without mdevs gets the empty
// document, like an accelerator class without devices.
Error Plugin::generateMdevCDISpec(const std::string &format) {
    mdevCdiFiles.clear();
    if (vgpuClasses.empty()) return Error();
    const int32_t fmt = format == "YAML" ? KXPU_FMT_YAML : KXPU_FMT_JSON;
    std::vector<size_t> entryClass;
    for (const auto &s : mdevState) entryClass.push_back(s.klass);
    return generateClassSpecs(vgpuClasses, mdevMap, entryClass, fmt, "kxpu_cdi_emit_mdev", emitMdevGroup, mdevCdiFiles);
}

// createDevicePlugins, device_plugin.go:83-112 (nothing is started: no gRPC here)
Error Plugin::createDevicePlugins() {
    std::vector<GenericDevicePlugin> dps;
    Error e = computeAer();  // the start-up walks are done: their AER counts
    if (e) return e;
    bool pt = false, vg = false;  // the first publication: generations stay 1
    updateAerTaints(pt, vg);
    e = buildPlugins(dps);
    devicePlugins.assign(std::make_move_iterator(dps.begin()), std::make_move_iterator(dps.end()));
    return e;
}

// the plugin list of the current maps, every device Healthy
Error Plugin::buildPlugins(std::vector<GenericDevicePlugin> &devicePlugins) {
    devicePlugins.clear();
    std::vector<std::string> ids, vendors;
    // position in names; a vfVgpu entry is named by its type key, an entry of a configured name by that name
    std::vector<size_t> nameAt(deviceMap.size(), 0);
    for (size_t d = 0; d < deviceMap.size(); d++) {
        const XpuClass &k = xpuClasses[d < deviceClass.size() ? deviceClass[d] : 0];
        if (k.vfVgpu || (d < deviceNamed.size() && deviceNamed[d])) continue;
        nameAt[d] = ids.size();
        ids.push_back(deviceMap[d].first);
        vendors.push_back(k.vendor);
    }
    std::map<std::string, size_t> modelAt;  // group of a class with resourceNames -> position of its model name in names
    for (size_t g = 0; g < iommuMap.size(); g++) {
        const GroupState<kxpu_dradev> &s = iommuState[g];
        if (xpuClasses[s.klass].resourceNames.empty()) continue;
        modelAt[iommuMap[g].first] = ids.size();
        ids.push_back(s.firstDevice);
        vendors.push_back(xpuClasses[s.klass].vendor);
    }
    const std::vector<std::string> names = getDeviceNames(ids, vendors);  // :99 for every device id at once
    // the Device of group id of a walk, Healthy, with the group's state
    auto device = [](const std::string &id, const std::map<std::string, size_t> &at, const auto &state) {
        Device d{id, kHealthy};
        auto it = at.find(id);
        if (it == at.end()) return d;
        const auto &s = state[it->second];
        d.numa = s.numa;
        d.pcieNode = s.pcieNode;
        d.blocker = s.blocker;
        d.aer = s.aer;
        return d;
    };
    const std::map<std::string, size_t> iommuAt = positions(iommuMap), mdevAt = positions(mdevMap);
    // a class with resourceNames: (class, final name) -> its plugin, which takes every entry of that name
    std::map<std::pair<size_t, std::string>, size_t> namedAt;
    std::set<size_t> merged;  // plugins that took a second entry: their groups go back to walk order
    size_t at = 0;
    for (const auto &kv : deviceMap) {  // :91
        GenericDevicePlugin dp;
        dp.xpuClass = at < deviceClass.size() ? deviceClass[at] : 0;
        dp.resourceNamespace = xpuClasses[dp.xpuClass].resourceNamespace;
        const bool renamed = !xpuClasses[dp.xpuClass].resourceNames.empty();
        for (const std::string &dev : kv.second) {  // :93-98
            dp.devs.push_back(device(dev, iommuAt, iommuState));
            auto m = modelAt.find(dev);
            if (m != modelAt.end()) dp.devs.back().model = names[m->second].empty() ? ids[m->second] : names[m->second];
        }
        const bool configured = at < deviceNamed.size() && deviceNamed[at];
        std::string devpluginName = xpuClasses[dp.xpuClass].vfVgpu || configured ? kv.first : names[nameAt[at]];
        at++;
        if (devpluginName.empty()) {
            fprintf(stderr, "Error: Could not find device name for device id: %s\n", kv.first.c_str());
            devpluginName = kv.first;  // :100-103
        }
        if (renamed) {
            auto it = namedAt.find({dp.xpuClass, devpluginName});
            if (it != namedAt.end()) {
                GenericDevicePlugin &into = devicePlugins[it->second];
                for (Device &d : dp.devs) into.devs.push_back(std::move(d));
                if (xpuClasses[dp.xpuClass].vfioCdev)
                    for (const auto &g : iommuMap) {
                        if (std::find(kv.second.begin(), kv.second.end(), g.first) == kv.second.end()) continue;
                        std::vector<std::string> &nodes = into.nodes[g.first];
                        for (const NvidiaGpuDevice &d : g.second)
                            if (d.cdev >= 0) nodes.push_back("vfio" + std::to_string(d.cdev));
                    }
                merged.insert(it->second);
                continue;
            }
            namedAt[{dp.xpuClass, devpluginName}] = devicePlugins.size();
        }
        dp.devpluginName = devpluginName;
        dp.devicePath = "/dev/vfio/";                                                          // :105
        if (xpuClasses[dp.xpuClass].vfioCdev) {  // every member's cdev node
            dp.devicePath = "/dev/vfio/devices/";
            for (const auto &g : iommuMap) {
                if (std::find(kv.second.begin(), kv.second.end(), g.first) == kv.second.end()) continue;
                std::vector<std::string> &nodes = dp.nodes[g.first];
                for (const NvidiaGpuDevice &d : g.second)
                    if (d.cdev >= 0) nodes.push_back("vfio" + std::to_string(d.cdev));
            }
        }
        dp.socketPath = std::string(kDevicePluginPath) + "kata-xpu-" + devpluginName + ".sock";  // generic:76
        dp.deviceKey = renamed ? devpluginName : kv.first;
        devicePlugins.push_back(std::move(dp));
    }
    for (size_t k : merged)
        std::stable_sort(devicePlugins[k].devs.begin(), devicePlugins[k].devs.end(), [&](const Device &a, const Device &b) {
            return iommuAt.at(a.ID) < iommuAt.at(b.ID);
        });
    for (size_t t = 0; t < typeMap.size(); t++) {  // one plugin per (vGPU class, type key)
        GenericDevicePlugin dp;
        dp.vgpu = true;
        dp.xpuClass = typeClass[t];
        dp.resourceNamespace = vgpuClasses[dp.xpuClass].resourceNamespace;
        for (const std::string &g : typeMap[t].second) dp.devs.push_back(device(g, mdevAt, mdevState));
        dp.devpluginName = typeMap[t].first;
        dp.devicePath = "/dev/vfio/";  // an mdev has its own IOMMU group and /dev/vfio/<group>
        if (vgpuClasses[dp.xpuClass].mdevCdev) {  // every mdev's cdev node
            dp.devicePath = "/dev/vfio/devices/";
            for (const auto &g : mdevMap) {
                const std::vector<std::string> &groups = typeMap[t].second;
                if (std::find(groups.begin(), groups.end(), g.first) == groups.end()) continue;
                std::vector<std::string> &nodes = dp.nodes[g.first];
                for (const MdevDevice &m : g.second)
                    if (m.cdev >= 0) nodes.push_back("vfio" + std::to_string(m.cdev));
            }
        }
        dp.socketPath = std::string(kDevicePluginPath) + "kata-xpu-" + dp.devpluginName + ".sock";
        dp.deviceKey = typeMap[t].first;
        devicePlugins.push_back(std::move(dp));
    }
    return Error();
}

bool Plugin::draEnabled() const {
    for (const XpuClass &c : xpuClasses)
        if (!c.draDriver.empty()) return true;
    return false;
}

bool Plugin::vfVgpuDraEnabled() const {
    for (const XpuClass &c : xpuClasses)
        if (!c.vgpuDraDriver.empty()) return true;
    return false;
}

bool Plugin::vgpuDraEnabled() const {
    for (const XpuClass &c : vgpuClasses)
        if (!c.draDriver.empty()) return true;
    return false;
}

// DRA drivers (draDriver and vgpuDraDriver) are distinct across xpuClasses and vgpuClasses (a passthrough class is named
// by its position, a vGPU class by "vGPU <position>", a vgpuDraDriver by its class's name and " vGPUs"), and a node name
// is required when any class has one
Error Plugin::checkDraClasses() const {
    std::vector<std::pair<const std::string *, std::string>> all;  // (driver, class name)
    for (size_t c = 0; c < xpuClasses.size(); c++) all.emplace_back(&xpuClasses[c].draDriver, std::to_string(c));
    for (size_t c = 0; c < vgpuClasses.size(); c++) all.emplace_back(&vgpuClasses[c].draDriver, "vGPU " + std::to_string(c));
    for (size_t c = 0; c < xpuClasses.size(); c++) all.emplace_back(&xpuClasses[c].vgpuDraDriver, std::to_string(c) + " vGPUs");
    for (size_t c = 0; c < vgpuClasses.size(); c++)
        all.emplace_back(&vgpuClasses[c].vgpuDraDriver, "vGPU " + std::to_string(c) + " vGPUs");
    for (size_t c = 0; c < all.size(); c++) {
        const std::string &d = *all[c].first;
        if (d.empty()) continue;
        if (nodeName.empty()) return fail("DRA driver " + d + " is set but the node name is empty (NODE_NAME)");
        for (size_t k = 0; k < c; k++)
            if (*all[k].first == d) return fail("DRA driver " + d + " is set on two classes (" + all[k].second + " and " + all[c].second + ")");
    }
    return Error();
}

Error Plugin::InitiateDevicePlugin() {
    Error e = checkDraClasses();
    if (!e) e = checkVfVgpuClasses();
    if (!e) e = checkResourceNames();
    if (!e) e = checkResetMethods();
    if (!e && vgpuSriovAware && vgpuClasses.empty()) e = fail("vgpuSriovAware is set but no vGPU class is configured");
    if (!e && sriovPfAware && !sriovAware) e = fail("sriovPfAware is set but sriovAware is off");
    if (!e && aerPortHealth && !aerHealth) e = fail("aerPortHealth is set but aerHealth is off");
    if (!e) e = checkDraPcieDomain();
    if (!e) e = checkDraVgpuPcie();
    if (e) return e;
    e = createIommuDeviceMap();  // :46
    if (e) return e;
    e = createMdevMap();
    if (e) return e;
    if (resumeIndices) {  // the state file first, then the specs, atomically and only when their bytes changed
        e = writeIndexState(&resume_.filesWritten);
        if (e) return e;
        atomicSpecs_ = true;
        specsWritten_.clear();
    }
    e = generateCDISpec(iommuMap);  // :49
    if (!e) e = generateMdevCDISpec();
    if (resumeIndices) {
        atomicSpecs_ = false;
        resume_.filesWritten.insert(resume_.filesWritten.end(), specsWritten_.begin(), specsWritten_.end());
    }
    if (e) return e;
    return createDevicePlugins();  // :52
}

// ---------------------------------------------------------------------------- restart resume (resumeIndices)
std::string formatIndexState(uint64_t pciNext, uint64_t mdevNext) {
    return "pci " + std::to_string(pciNext) + "\nmdev " + std::to_string(mdevNext) + "\n";
}

// a canonical decimal below 2^64
static bool parseU64(const std::string &s, uint64_t &v) {
    if (s.empty() || s.size() > 20 || (s.size() > 1 && s[0] == '0')) return false;
    uint64_t x = 0;
    for (char c : s) {
        if (c < '0' || c > '9') return false;
        const uint64_t d = (uint64_t)(c - '0');
        if (x > (UINT64_MAX - d) / 10) return false;
        x = x * 10 + d;
    }
    v = x;
    return true;
}

bool parseIndexState(const std::string &text, uint64_t &pciNext, uint64_t &mdevNext) {
    const size_t nl = text.find('\n');
    if (text.compare(0, 4, "pci ") != 0 || nl == std::string::npos || text.compare(nl + 1, 5, "mdev ") != 0) return false;
    const size_t nl2 = text.find('\n', nl + 1);
    if (nl2 == std::string::npos || nl2 + 1 != text.size()) return false;
    uint64_t p = 0, m = 0;
    if (!parseU64(text.substr(4, nl - 4), p) || !parseU64(text.substr(nl + 6, nl2 - nl - 6), m)) return false;
    pciNext = p;
    mdevNext = m;
    return true;
}

static const char *kIndexStateName = ".kata-xpu-cdi-index";  // not *.json / *.yaml: the CDI cache ignores it

static bool readWholeFile(const std::string &path, std::string &out, bool &missing) {
    missing = false;
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) { missing = errno == ENOENT; return false; }
    out.clear();
    char buf[1 << 16];
    size_t k;
    while ((k = fread(buf, 1, sizeof buf, f)) > 0) out.append(buf, k);
    const bool ok = !ferror(f);
    fclose(f);
    return ok;
}

void Plugin::readIndexState() {
    const std::string path = cdiConfigPath + kIndexStateName;
    std::string text;
    bool missing = false;
    if (!readWholeFile(path, text, missing)) {
        if (!missing) fprintf(stderr, "CDI index state %s: unreadable (%s), resuming without it\n", path.c_str(), strerror(errno));
        return;
    }
    resume_.stateRead = parseIndexState(text, resume_.statePci, resume_.stateMdev);
    if (!resume_.stateRead) fprintf(stderr, "CDI index state %s: malformed, resuming without it\n", path.c_str());
}

Error Plugin::writeIndexState(std::vector<std::string> *written) {
    const std::string path = cdiConfigPath + kIndexStateName;
    const std::string text = formatIndexState(pci_.next, mdev_.next);
    bool w = false;
    Error e = writeSpecFileAtomic(path, reinterpret_cast<const uint8_t *>(text.data()), text.size(), w);
    if (w && written) written->push_back(path);
    return e;
}

template <typename Rec>
void Plugin::previousEntries(const std::vector<XpuClass> &classes,
                             int32_t (*parse)(kxpu_ctx *, int32_t, const char *, const uint8_t *, size_t, Rec *, size_t, size_t *),
                             uint64_t stateNext, ResumeWalk &rw, std::vector<kxpu_snaprec> &prev, uint64_t &next) {
    prev.clear();
    next = stateNext;
    std::set<std::string> keys;
    std::set<uint64_t> indices;
    for (size_t c = 0; c < classes.size() && rw.fallback.empty(); c++) {
        const std::string path = cdiConfigPath + classes[c].cdiFileStem + ".yaml";
        std::string doc;
        bool missing = false;
        if (!readWholeFile(path, doc, missing)) {
            if (!missing) rw.fallback = path + ": unreadable: " + strerror(errno);
            continue;  // a missing file holds no entries
        }
        std::vector<Rec> recs(doc.size() / KXPU_CDI_FRAG_MIN + 1);
        size_t n = 0;
        auto parseWith = [&](decltype(parse) fn) {
            return fn(ctx_, KXPU_FMT_YAML, classes[c].cdiKind.c_str(), reinterpret_cast<const uint8_t *>(doc.data()), doc.size(),
                      recs.data(), recs.size(), &n);
        };
        int32_t rc;
        bool typed = false;  // each entry's vGPU type was read back
        if constexpr (std::is_same<Rec, kxpu_vfvgpucdi>::value) {
            // the layout the class uses now, then the other one; a vfVgpu class tries its typed layouts first
            rc = KXPU_E_INVALID;
            if (classes[c].vfVgpu) {
                rc = parseWith(classes[c].vfioCdev ? kxpu_cdi_parse_vf_vgpu_cdev : kxpu_cdi_parse_vf_vgpu);
                if (rc == KXPU_E_INVALID) rc = parseWith(classes[c].vfioCdev ? kxpu_cdi_parse_vf_vgpu : kxpu_cdi_parse_vf_vgpu_cdev);
                typed = rc != KXPU_E_INVALID;
            }
            if (rc == KXPU_E_INVALID) rc = parseWith(classes[c].vfioCdev ? parsePciCdev : parsePciGroup);
            if (rc == KXPU_E_INVALID) rc = parseWith(classes[c].vfioCdev ? parsePciGroup : parsePciCdev);
        } else {
            rc = parseWith(classes[c].mdevCdev ? kxpu_cdi_parse_mdev_cdev : parse);
            if (rc == KXPU_E_INVALID) rc = parseWith(classes[c].mdevCdev ? parse : kxpu_cdi_parse_mdev_cdev);
        }
        if (rc != KXPU_OK) {
            rw.fallback = path + ": not a CDI spec this plugin writes (" + kxpu_strerror(rc) + ": " + kxpu_last_error(ctx_) + ")";
            break;
        }
        rw.filesRead.push_back(path);
        if constexpr (std::is_same<Rec, kxpu_vfvgpucdi>::value) {
            if (typed) {  // the names of the types the spec lists, for the walk's type join: the first key of an ID wins
                rw.typedClasses.insert(c);
                for (size_t i = 0; i < n; i++) {
                    const std::string key(recs[i].key, recs[i].key_len);
                    auto it = learnedVgpuTypes_.emplace(recs[i].type_id, key).first;
                    if (it->second != key)
                        fprintf(stderr, "%s: vGPU type %u is named %s here and %s before; keeping %s\n", path.c_str(),
                                recs[i].type_id, key.c_str(), it->second.c_str(), it->second.c_str());
                }
            }
        }
        for (size_t i = 0; i < n && rw.fallback.empty(); i++) {
            const auto &r = cdiBase(recs[i]);
            kxpu_snaprec s;
            memset(&s, 0, sizeof s);
            if constexpr (std::is_same<Rec, kxpu_mdevcdev>::value) memcpy(s.key, r.uuid, sizeof r.uuid);
            else memcpy(s.key, r.bdf, strnlen(r.bdf, sizeof r.bdf));
            s.iommu_group = r.iommu_group;
            s.klass = (uint32_t)c;
            s.index = r.index;
            // a typed entry carries the tag snapshotOf gives a vGPU VF: a VF whose type changed gets a fresh index
            if constexpr (std::is_same<Rec, kxpu_vfvgpucdi>::value)
                if (typed) s.tag = 1ull << 63 | recs[i].type_id;
            const std::string key(s.key, strnlen(s.key, sizeof s.key));
            if (r.index == UINT64_MAX) rw.fallback = path + ": index 18446744073709551615";
            else if (!indices.insert(r.index).second) rw.fallback = path + ": index " + std::to_string(r.index) + " named twice";
            else if (!keys.insert(key).second) rw.fallback = path + ": " + key + " named twice";
            else {
                prev.push_back(s);
                next = std::max(next, r.index + 1);
            }
        }
    }
}

Error Plugin::resumeWalk(std::vector<kxpu_snaprec> prev, uint64_t next, uint64_t stateNext, const std::vector<kxpu_snaprec> &cur,
                         ResumeWalk &rw, std::vector<uint64_t> &index, uint64_t &nextOut) {
    index.assign(cur.size() + 1, 0);
    for (int attempt = 0; attempt < 2; attempt++) {
        if (!rw.fallback.empty()) {  // nothing known: fresh indices above everything the state file says was handed out
            fprintf(stderr, "CDI index resume: %s; numbering this walk afresh from %llu\n", rw.fallback.c_str(),
                    (unsigned long long)stateNext);
            prev.clear();
            next = stateNext;
        }
        const int32_t rc = kxpu_reconcile(ctx_, prev.data(), prev.size(), next, cur.data(), cur.size(), index.data(), nullptr,
                                          nullptr, &rw.counts);
        if (rc == KXPU_OK) break;
        if (rc != KXPU_E_INVALID || !rw.fallback.empty()) return kxfail(ctx_, "kxpu_reconcile", rc);
        rw.fallback = std::string("kxpu_reconcile refused the previous entries: ") + kxpu_last_error(ctx_);
    }
    index.resize(cur.size());
    nextOut = rw.counts.next_index_out;
    return Error();
}

template <typename Walk>
Error Plugin::resume(const Walk &w, WalkBook &book, ResumeWalk &rw, uint64_t stateNext, std::vector<kxpu_snaprec> prev,
                     uint64_t next) {
    std::vector<kxpu_snaprec> cur = snapshotOf(w, nullptr);
    std::map<uint32_t, size_t> groupClass = groupClasses(w.out);  // the file generateClassSpecs puts the entry in
    // tag 0, but a vGPU VF of a class whose spec was read typed keeps its type tag, as the entries read from that spec do
    for (kxpu_snaprec &s : cur) {
        s.klass = (uint32_t)groupClass[s.iommu_group];
        if (!(rw.typedClasses.count(s.klass) && (s.tag >> 63))) s.tag = 0;
    }
    std::vector<uint64_t> index;
    Error e = resumeWalk(std::move(prev), next, stateNext, cur, rw, index, book.next);
    if (e) return e;
    buildMaps(w, &index);
    book.snap = snapshotOf(w, &index);
    return Error();
}

bool Plugin::discoveryStale() {
    return !(pci_.current(bindGeneration) && (vgpuClasses.empty() || mdev_.current(mdevGeneration)));
}

template <typename Walk>
Error Plugin::rewalk(Walk &w, WalkBook &book, kxpu_reconcile_counts &counts) {
    Error e = classify(w);
    if (e) return e;
    const std::vector<kxpu_snaprec> cur = snapshotOf(w, nullptr);
    std::vector<uint64_t> index(cur.size() + 1, 0);
    const int32_t rc = kxpu_reconcile(ctx_, book.snap.data(), book.snap.size(), book.next, cur.data(), cur.size(), index.data(),
                                      nullptr, nullptr, &counts);
    if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_reconcile", rc);
    index.resize(cur.size());
    book.snap = cur;
    for (size_t i = 0; i < book.snap.size(); i++) book.snap[i].index = index[i];
    book.next = counts.next_index_out;
    buildMaps(w, &index);
    return Error();
}

Error Plugin::rediscover(RediscoverReport &report, const std::string &format) {
    std::unique_lock<std::shared_mutex> lock(mu_);
    report = RediscoverReport();
    report.pci.next_index_out = pci_.next;
    report.mdev.next_index_out = mdev_.next;
    // 1. the generations BEFORE the walks (an event during a walk makes the result stale, never fresh)
    uint64_t gen = 0, mgen = 0;
    const bool haveGen = bindGeneration && bindGeneration(gen);
    const bool haveMgen = !vgpuClasses.empty() && mdevGeneration && mdevGeneration(mgen);
    // 2.-3. the same walks and classify variants as start-up, reconciled against the snapshots
    std::map<std::string, std::string> blockerWas;  // group id -> its blocker in the last walk
    for (size_t g = 0; g < iommuMap.size(); g++) blockerWas[iommuMap[g].first] = iommuState[g].blocker;
    std::map<std::string, std::pair<std::string, std::string>> pfWas;  // sriovPfAware: group id -> its PF and PF device id
    for (size_t g = 0; sriovPfAware && g < iommuMap.size(); g++)
        pfWas[iommuMap[g].first] = {iommuState[g].pf, iommuState[g].pfDevice};
    std::map<std::string, std::pair<uint64_t, uint64_t>> portsWas;  // draPcieDomain: group id -> its root port and switch
    for (size_t g = 0; !draPcieDomain.empty() && g < iommuMap.size(); g++)
        portsWas[iommuMap[g].first] = {iommuState[g].rootPort, iommuState[g].pcieSwitch};
    PciWalk pw;
    Error e = rewalk(pw, pci_, report.pci);
    if (e) return e;
    bool viabilityChanged = false, pfChanged = false, portsChanged = false;
    for (size_t g = 0; g < iommuMap.size(); g++) {
        auto it = blockerWas.find(iommuMap[g].first);
        viabilityChanged |= it != blockerWas.end() && it->second != iommuState[g].blocker;
        auto pt = pfWas.find(iommuMap[g].first);  // a VF whose PF changed is published with other attributes
        pfChanged |= pt != pfWas.end() && pt->second != std::make_pair(iommuState[g].pf, iommuState[g].pfDevice);
        auto qt = portsWas.find(iommuMap[g].first);  // a device moved under another root port or switch
        portsChanged |= qt != portsWas.end() && qt->second != std::make_pair(iommuState[g].rootPort, iommuState[g].pcieSwitch);
    }
    std::map<std::string, std::pair<uint64_t, uint64_t>> mdevPortsWas;  // draVgpuPcie: mdev group id -> its ports
    for (size_t g = 0; draVgpuPcie && g < mdevMap.size(); g++)
        mdevPortsWas[mdevMap[g].first] = {mdevState[g].rootPort, mdevState[g].pcieSwitch};
    bool mdevPortsChanged = false;
    if (!vgpuClasses.empty()) {
        MdevWalk mw;
        e = rewalk(mw, mdev_, report.mdev);
        if (e) return e;
        for (size_t g = 0; g < mdevMap.size(); g++) {  // a vGPU moved under another root port or switch
            auto qt = mdevPortsWas.find(mdevMap[g].first);
            mdevPortsChanged |= qt != mdevPortsWas.end() &&
                                qt->second != std::make_pair(mdevState[g].rootPort, mdevState[g].pcieSwitch);
        }
    }
    e = computeAer();  // a re-enumerated function starts with zeroed counters
    if (e) return e;
    if (resumeIndices) {  // the next indices reach the state file before any spec names one of them
        e = writeIndexState(nullptr);
        if (e) return e;
    }
    // 4. the CDI specs: a file is rewritten only when its bytes changed, atomically
    atomicSpecs_ = true;
    specsWritten_.clear();
    e = generateCDISpec(iommuMap, format);
    if (!e) e = generateMdevCDISpec(format);
    atomicSpecs_ = false;
    report.cdiFilesWritten = specsWritten_;
    if (e) return e;
    // 5. devicePlugins in place: health carried per group, new groups Healthy, new plugins appended
    std::vector<GenericDevicePlugin> want;
    e = buildPlugins(want);
    if (e) return e;
    std::map<std::string, std::string> healthOf;
    for (const GenericDevicePlugin &dp : devicePlugins)
        for (const Device &d : dp.devs) healthOf[d.ID] = d.Health;
    std::vector<bool> seen(devicePlugins.size(), false);
    for (GenericDevicePlugin &w : want) {
        for (Device &d : w.devs) {
            auto it = healthOf.find(d.ID);
            if (it != healthOf.end()) d.Health = it->second;
        }
        size_t at = devicePlugins.size();
        for (size_t k = 0; k < devicePlugins.size(); k++) {
            const GenericDevicePlugin &o = devicePlugins[k];
            if (!seen[k] && o.vgpu == w.vgpu && o.xpuClass == w.xpuClass && o.deviceKey == w.deviceKey) { at = k; break; }
        }
        if (at == devicePlugins.size()) {
            devicePlugins.push_back(std::move(w));
            seen.push_back(true);
            report.addedPlugins.push_back(at);
            report.changedPlugins.push_back(at);
            continue;
        }
        seen[at] = true;
        std::vector<Device> &cur = devicePlugins[at].devs;
        bool same = cur.size() == w.devs.size();
        for (size_t i = 0; same && i < cur.size(); i++)
            same = cur[i].ID == w.devs[i].ID && cur[i].Health == w.devs[i].Health && cur[i].numa == w.devs[i].numa &&
                   cur[i].pcieNode == w.devs[i].pcieNode && cur[i].blocker == w.devs[i].blocker && cur[i].aer == w.devs[i].aer &&
                   cur[i].drift == w.devs[i].drift && cur[i].model == w.devs[i].model;
        if (!same || devicePlugins[at].nodes != w.nodes) {  // changed cdev nodes: the watcher must follow them
            cur = std::move(w.devs);
            devicePlugins[at].nodes = std::move(w.nodes);
            report.changedPlugins.push_back(at);
        }
    }
    for (size_t k = 0; k < seen.size(); k++) {
        if (seen[k] || devicePlugins[k].devs.empty()) continue;
        devicePlugins[k].devs.clear();  // every device left: the resource stays, with an empty list
        report.changedPlugins.push_back(k);
    }
    std::sort(report.changedPlugins.begin(), report.changedPlugins.end());
    // a surviving group keeps its taint time, as it keeps its health; a group that left drops it
    for (auto it = draTaintSince_.begin(); it != draTaintSince_.end();) {
        bool present = false;
        for (const auto &kv : iommuMap) present |= kv.first == it->first;
        for (const auto &kv : mdevMap) present |= kv.first == it->first;
        it = present ? std::next(it) : draTaintSince_.erase(it);
    }
    bool passthroughChanged = false, vgpuChanged = false;
    for (size_t k : report.changedPlugins) (devicePlugins[k].vgpu ? vgpuChanged : passthroughChanged) = true;
    bool aerPt = false, aerVg = false;
    updateAerTaints(aerPt, aerVg);
    const bool driftCleared = !driftTaint_.empty();  // the walk is the new truth: every drift reason is gone
    driftTaint_.clear();
    if (passthroughChanged || viabilityChanged || pfChanged || portsChanged || aerPt || driftCleared) pci_.draGeneration++;  // the next publication replaces these slices
    if (vgpuChanged || mdevPortsChanged || aerVg) mdev_.draGeneration++;
    // 6. a fresh snapshot generation: Allocate answers from the snapshot again
    pci_.haveGen = haveGen;
    pci_.gen = gen;
    mdev_.haveGen = haveMgen;
    mdev_.gen = mgen;
    haveSnapshotGen_ = snapshotValidation && haveGen;
    snapshotGen_ = gen;
    return Error();
}

// kxpu_sriov's canonical PCI address: "dddd:bb:dd.f", lowercase hex, device at most 1f, function 0..7
static bool canonicalBdf(const std::string &a) {
    if (a.size() != 12 || a[4] != ':' || a[7] != ':' || a[10] != '.' || a[11] < '0' || a[11] > '7' || a[8] > '1') return false;
    for (int k : {0, 1, 2, 3, 5, 6, 8, 9})
        if (!((a[k] >= '0' && a[k] <= '9') || (a[k] >= 'a' && a[k] <= 'f'))) return false;
    return true;
}

// kxpu_sriov's sriov_numvfs rule: at most one trailing '\n', then a canonical decimal 0..65535; anything else 0
static uint32_t parseNumvfs(const kxpu_sriovrec &s) {
    if ((s.flags & KXPU_SR_NUMVFS_ERR) || s.numvfs_len > sizeof s.numvfs_txt) return 0;
    std::string t((const char *)s.numvfs_txt, s.numvfs_len);
    if (!t.empty() && t.back() == '\n') t.pop_back();
    if (t.empty() || t.size() > 5 || (t.size() > 1 && t[0] == '0')) return 0;
    uint32_t v = 0;
    for (char ch : t) {
        if (ch < '0' || ch > '9') return 0;
        v = v * 10 + (uint32_t)(ch - '0');
    }
    return v <= 65535 ? v : 0;
}

std::string Plugin::sriovLive(const std::string &bdf) {
    const kxpu_sriovrec s = readSriov(bdf);
    const std::string pf(s.physfn, strnlen(s.physfn, sizeof s.physfn));
    if (!(s.flags & KXPU_SR_PHYSFN_ERR) && canonicalBdf(pf) && pf != bdf) {
        char buf[4096];
        const ssize_t n = readlink((basePath + "/" + pf + "/driver").c_str(), buf, sizeof buf - 1);
        if (n >= 0) {
            const std::string target(buf, (size_t)n);
            const std::string drv = target.substr(target.find_last_of('/') + 1);  // npos + 1 == 0
            if (passthroughDriver(drv)) return sriovVfReason(bdf, pf, drv);
        }
    }
    const uint32_t k = parseNumvfs(s);
    return k ? sriovPfReason(bdf, k) : std::string();
}

// kxpu_vf_vgpu_types' current-type rule: at most one trailing '\n', then a canonical decimal below 2^32; 0 for anything
// else (no vGPU, or not a type ID)
static uint32_t parseVgpuType(std::string t) {
    if (!t.empty() && t.back() == '\n') t.pop_back();
    if (t.empty() || t.size() > 10 || (t.size() > 1 && t[0] == '0')) return 0;
    uint64_t v = 0;
    for (char ch : t) {
        if (ch < '0' || ch > '9') return 0;
        v = v * 10 + (uint64_t)(ch - '0');
    }
    return v < (1ull << 32) ? (uint32_t)v : 0;
}

// Allocate, generic_device_plugin.go:320-355, for one ContainerAllocateRequest
Error Plugin::Allocate(const std::vector<std::string> &devicesIDs, ContainerAllocateResponse &resp) {
    std::shared_lock<std::shared_mutex> lock(mu_);  // a rediscovery rebuilds the maps under the exclusive lock
    std::vector<uint64_t> devIndexes;
    const auto &returnedMap = returnIommuMap();
    // snapshot validation (off by default): every device of returnedMap was NVIDIA, bound to vfio-pci and in
    // this group when it was discovered; if no pci function was bound / unbound / added / removed since, the
    // live reads below would return exactly that
    bool fromSnapshot = false;
    if (snapshotValidation && haveSnapshotGen_ && bindGeneration) {
        uint64_t now = 0;
        fromSnapshot = bindGeneration(now) && now == snapshotGen_;
    }
    size_t reqClass = 0;  // the class of the request's groups: one plugin serves one class
    const auto &mdevs = returnMdevMap();
    bool havePci = false, haveVgpu = false;
    size_t vgpuClass = 0;
    for (const std::string &iommuId : devicesIDs) {  // :324
        const std::vector<MdevDevice> *mDevs = nullptr;
        for (const auto &kv : mdevs) if (kv.first == iommuId) { mDevs = &kv.second; break; }
        if (mDevs) {  // a vGPU group: always live reads (the uevent snapshot only follows PCI binds)
            const GroupState<kxpu_dramdev> *s = stateOf(mdevMap, mdevState, iommuId);
            if (s && !s->blocker.empty())  // the verdict of the last walk, before any read
                return fail("invalid allocation request: IOMMU group " + iommuId + " is not viable: " + s->blocker);
            const size_t c = s ? s->klass : 0;
            if (havePci || (haveVgpu && c != vgpuClass)) return fail("invalid allocation request: devices of more than one class");
            haveVgpu = true;
            vgpuClass = c;
            for (const MdevDevice &m : *mDevs) {
                liveValidations++;
                std::string iommuGroup, vendor;
                if (!readLink(mdevBasePath, m.uuid, "iommu_group", iommuGroup) || iommuGroup != iommuId ||
                    !readIDFromFile(mdevBasePath, m.uuid, "../vendor", vendor) || trimID(vendor) != vgpuClasses[m.vgpuClass].vendor)
                    return fail("invalid allocation request: unknown device: " + m.uuid);
                if (vgpuClasses[c].mdevCdev && readVfioCdev(mdevBasePath, m.uuid) != m.cdev)  // numbers are reused
                    return fail("invalid allocation request: the VFIO cdev of " + m.uuid + " changed since discovery");
                devIndexes.push_back(m.index);
            }
            continue;
        }
        const std::vector<NvidiaGpuDevice> *nvDevs = nullptr;
        for (const auto &kv : returnedMap) if (kv.first == iommuId) { nvDevs = &kv.second; break; }
        if (!nvDevs) continue;  // unknown group id: empty nvDevs, no error (:327)
        const GroupState<kxpu_dradev> *s = stateOf(iommuMap, iommuState, iommuId);
        if (s && !s->blocker.empty())  // the verdict of the last walk, before any read
            return fail("invalid allocation request: IOMMU group " + iommuId + " is not viable: " + s->blocker);
        const size_t c = s ? s->klass : 0;
        if (haveVgpu || (havePci && c != reqClass)) return fail("invalid allocation request: devices of more than one class");
        havePci = true;
        reqClass = c;
        for (const NvidiaGpuDevice &dev : *nvDevs) {
            if (fromSnapshot && !xpuClasses[c].vfVgpu) {  // a type change sends no uevent: a vGPU VF is always re-read
                snapshotValidations++;
                devIndexes.push_back(dev.index);  // :340
                continue;
            }
            liveValidations++;
            std::string iommuGroup, vendor;
            if (!readLink(basePath, dev.addr, "iommu_group", iommuGroup) || iommuGroup != iommuId)  // :329-333
                return fail("invalid allocation request: unknown device: " + dev.addr);
            const std::string &want = xpuClasses[dev.xpuClass].vendor;  // the device's class
            if (!readIDFromFile(basePath, dev.addr, "vendor", vendor) || trimID(vendor) != want)  // :334-338
                return fail("invalid allocation request: unknown device: " + dev.addr);
            if (xpuClasses[c].vfioCdev && readVfioCdev(basePath, dev.addr) != dev.cdev)  // cdev numbers are reused across re-binds
                return fail("invalid allocation request: the VFIO cdev of " + dev.addr + " changed since discovery");
            if (xpuClasses[c].vfVgpu) {  // the profile the walk saw, or the CDI index names another vGPU now
                std::string cur;
                const uint32_t now = readVgpuFile(basePath, dev.addr, "current_vgpu_type", cur) ? parseVgpuType(cur) : 0;
                vfVgpuReads++;
                if (now != dev.vgpuType)
                    return fail("invalid allocation request: " + dev.addr + " carries vGPU type " + std::to_string(now) +
                                ", not type " + std::to_string(dev.vgpuType) + " as discovered");
            }
            if (sriovAware) {  // a PF rebound, or VFs enabled, since the walk
                const std::string why = sriovLive(dev.addr);
                if (!why.empty()) return fail("invalid allocation request: " + why);
            }
            devIndexes.push_back(dev.index);  // :340
        }
    }
    const std::string &kind = haveVgpu ? vgpuClasses[vgpuClass].cdiKind : xpuClasses[reqClass].cdiKind;
    resp.CDIDevices.clear();
    if (!devIndexes.empty()) {  // updateResponseForCDI :274-299; strategy cdi-cri is on (:61)
        std::vector<uint32_t> offs(devIndexes.size() + 1);
        size_t need = 0;
        std::vector<uint8_t> buf((kind.size() + 22) * devIndexes.size());
        const int32_t rc =
            kxpu_alloc_names_kind(ctx_, kind.c_str(), devIndexes.data(), devIndexes.size(), buf.data(), buf.size(), offs.data(), &need);
        if (rc != KXPU_OK) return fail("failed to get allocate response: " + std::string(kxpu_strerror(rc)));
        for (size_t i = 0; i < devIndexes.size(); i++)
            resp.CDIDevices.emplace_back((const char *)buf.data() + offs[i], offs[i + 1] - offs[i]);
    }
    resp.Envs.clear();
    resp.Envs[kK8SCDIVendorClass] = kind;  // :348-350 overwrites Envs
    return Error();
}

// The taint of a group whose device node the HealthWatcher saw disappear.  The effect is NoSchedule on purpose: it keeps
// new claims away, and a missing /dev/vfio node must not evict a VM that already holds the group open, which NoExecute
// would do.
static const char *kDraTaintKeyName = "/unhealthy";  // the key is <draDriver>/unhealthy
static const char *kDraTaintValue = "vfio-device-missing";
static const char *kDraTaintEffect = "NoSchedule";

// With aerHealth, the table goes on with the AER taint's two values.  The two AER entries share key and effect, so a
// group carries at most one of them.
static const char *kAerTaintKeyName = "/pcie-aer";  // the key is <draDriver>/pcie-aer

// With vfVgpuHealth, a VF-vGPU pool's table has a fourth entry: the VF no longer carries the type it is published with.
static const char *kTypeTaintKeyName = "/vgpu-type";  // the key is <vgpuDraDriver>/vgpu-type
static const char *kTypeTaintValue = "changed";

// f(group id, state) for every group of a walk (map, states, the walk's class list) that is published in its class's
// pool, in walk order: the group has a ResourceSlice record, its class a draDriver, and it has no blocker.  Only a
// published group gets taints.
template <typename V, typename Dra, typename F>
static void forPublished(const OrderedMap<V> &m, const std::vector<GroupState<Dra>> &state, const std::vector<XpuClass> &classes,
                         F f) {
    for (size_t g = 0; g < m.size(); g++)
        if (state[g].dra && !classes[state[g].klass].draDriver.empty() && state[g].blocker.empty()) f(m[g].first, state[g]);
}
// the same for the VF-vGPU pools of the PCI walk: the group has a VF-vGPU record, its class a vgpuDraDriver, and it has
// no blocker
template <typename F>
static void forPublishedVfVgpu(const OrderedMap<std::vector<NvidiaGpuDevice>> &m, const std::vector<GroupState<kxpu_dradev>> &state,
                               const std::vector<XpuClass> &classes, F f) {
    for (size_t g = 0; g < m.size(); g++)
        if (state[g].vfVgpuDra && !classes[state[g].klass].vgpuDraDriver.empty() && state[g].blocker.empty())
            f(m[g].first, state[g]);
}

template <typename Rec, typename Fn>
Error Plugin::draSlices(Fn fn, const char *what, const std::string &driver, uint64_t generation, const std::vector<Rec> &devs,
                        const std::vector<std::string> &groups, std::vector<uint8_t> &out, std::vector<uint64_t> &sliceOff,
                        bool typeTaint) const {
    const std::string missing = driver + kDraTaintKeyName, aer = driver + kAerTaintKeyName, type = driver + kTypeTaintKeyName;
    const kxpu_dra_taint table[4] = {{missing.c_str(), kDraTaintValue, kDraTaintEffect},
                                     {aer.c_str(), "fatal", kDraTaintEffect},
                                     {aer.c_str(), "nonfatal", kDraTaintEffect},
                                     {type.c_str(), kTypeTaintValue, kDraTaintEffect}};
    const size_t nt = typeTaint ? 4 : aerHealth ? 3 : 1;
    const std::vector<int64_t> since = draTaints ? draSinceTable(groups, typeTaint) : std::vector<int64_t>();
    const int64_t *ts = draTaints ? since.data() : nullptr;  // NULL: the untainted slices
    size_t len = 0, nSlices = 0;
    int32_t rc = fn(ctx_, driver.c_str(), nodeName.c_str(), nodeName.c_str(), generation, devs.data(), devs.size(), table, nt,
                    ts, nullptr, 0, &len, nullptr, &nSlices);
    if (rc == KXPU_E_NOSPACE) {
        out.assign(len, 0);
        sliceOff.assign(nSlices + 1, 0);
        rc = fn(ctx_, driver.c_str(), nodeName.c_str(), nodeName.c_str(), generation, devs.data(), devs.size(), table, nt, ts,
                out.data(), out.size(), &len, sliceOff.data(), &nSlices);
    }
    if (rc != KXPU_OK) return kxfail(ctx_, what, rc);
    return Error();
}

Error Plugin::ResourceSlices(size_t xpuClass, std::vector<uint8_t> &out, std::vector<uint64_t> &sliceOff) {
    std::shared_lock<std::shared_mutex> lock(mu_);
    if (xpuClass >= xpuClasses.size() || xpuClasses[xpuClass].draDriver.empty())
        return fail("ResourceSlices: class " + std::to_string(xpuClass) + " has no DRA driver");
    // group id -> its model name: the resource-name suffix of its plugin, or with resourceNames the group's own
    std::map<std::string, const std::string *> productOf;
    for (const GenericDevicePlugin &dp : devicePlugins)
        if (!dp.vgpu && dp.xpuClass == xpuClass)
            for (const Device &d : dp.devs) productOf[d.ID] = d.model.empty() ? &dp.devpluginName : &d.model;
    std::vector<kxpu_dradev> devs;
    std::vector<kxpu_dradevpf> pfDevs;  // sriovPfAware: the same devices with their PFs
    std::vector<kxpu_dradevpcie> pcieDevs;  // draPcieDomain: the same devices with their PFs (sriovPfAware) and ports
    std::vector<std::string> groups;
    forPublished(iommuMap, iommuState, xpuClasses, [&](const std::string &g, const GroupState<kxpu_dradev> &s) {
        if (s.klass != xpuClass) return;
        kxpu_dradev d = *s.dra;
        auto it = productOf.find(g);
        if (it != productOf.end()) {
            d.product_len = (uint8_t)std::min<size_t>(it->second->size(), sizeof d.product);
            memcpy(d.product, it->second->data(), d.product_len);
        }
        groups.push_back(g);
        if (!sriovPfAware && draPcieDomain.empty()) {
            devs.push_back(d);
            return;
        }
        kxpu_dradevpf p;
        memset(&p, 0, sizeof p);
        p.dev = d;
        if (sriovPfAware) {
            memcpy(p.physfn, s.pf.data(), std::min(s.pf.size(), sizeof p.physfn));
            memcpy(p.physfn_device, s.pfDevice.data(), std::min(s.pfDevice.size(), sizeof p.physfn_device));
        }
        if (draPcieDomain.empty()) {
            pfDevs.push_back(p);
            return;
        }
        kxpu_dradevpcie q;
        memset(&q, 0, sizeof q);
        q.pf = p;
        q.root_port = s.rootPort;
        q.pcie_switch = s.pcieSwitch;
        pcieDevs.push_back(q);
    });
    if (!draPcieDomain.empty()) {
        const char *domain = draPcieDomain.c_str();
        auto fn = [domain](kxpu_ctx *ctx, const char *driver, const char *pool, const char *node, uint64_t generation,
                           const kxpu_dradevpcie *v, size_t n, const kxpu_dra_taint *taints, size_t nt, const int64_t *since,
                           uint8_t *o, size_t cap, size_t *len, uint64_t *off, size_t *ns) {
            return kxpu_dra_slices_pcie(ctx, driver, pool, node, generation, domain, v, n, taints, nt, since, o, cap, len,
                                        off, ns);
        };
        return draSlices(fn, "kxpu_dra_slices_pcie", xpuClasses[xpuClass].draDriver, pci_.draGeneration, pcieDevs, groups,
                         out, sliceOff);
    }
    if (sriovPfAware)
        return draSlices(kxpu_dra_slices_pf, "kxpu_dra_slices_pf", xpuClasses[xpuClass].draDriver, pci_.draGeneration,
                         pfDevs, groups, out, sliceOff);
    return draSlices(kxpu_dra_slices_taints, "kxpu_dra_slices_taints", xpuClasses[xpuClass].draDriver, pci_.draGeneration, devs,
                     groups, out, sliceOff);
}

std::vector<int64_t> Plugin::draSinceTable(const std::vector<std::string> &groups, bool typeTaint) const {
    std::vector<int64_t> since;
    for (const std::string &g : groups) {
        auto it = draTaintSince_.find(g);
        since.push_back(it == draTaintSince_.end() ? -1 : it->second);
        if (!aerHealth && !typeTaint) continue;
        auto at = aerTaint_.find(g);  // empty without aerHealth
        const uint8_t v = at == aerTaint_.end() ? 0 : at->second.first;
        since.push_back(v == KXPU_AER_FATAL ? at->second.second : -1);
        since.push_back(v == KXPU_AER_NONFATAL ? at->second.second : -1);
        if (!typeTaint) continue;
        auto dt = driftTaint_.find(g);
        since.push_back(dt == driftTaint_.end() ? -1 : dt->second);
    }
    return since;
}

Error Plugin::computeAer() {
    auto set = [](auto &s, const std::string &why, uint8_t bits) {
        s.aer = why;
        s.aerBits = bits;
        s.aerMax[0] = s.aerMax[1] = KXPU_METRICS_NO_VALUE;
    };
    for (auto &s : iommuState) set(s, std::string(), 0);
    for (auto &s : mdevState) set(s, std::string(), 0);
    if (!aerHealth) return Error();  // no aer_dev_* file is opened
    // one record per member of every group, passthrough groups then vGPU groups; a vGPU reads its parent's files.  With
    // vfVgpuHealth a group whose first member is a VF of a vfVgpu class, with sriovPfAware a group of another class whose
    // first member is a VF, and with vgpuSriovAware a vGPU group whose first mdev's parent is a VF, has its PF as one
    // more member, one record per PF.
    std::string text;
    std::vector<uint64_t> off;
    std::vector<uint32_t> len, goff{0}, members;
    std::vector<std::string> who;  // the function whose files record i read
    std::map<std::string, uint32_t> pfRecord;  // PF address -> its record
    // aerPortHealth: after a group's members and PF, the ports above its members, one record per port address shared by
    // every group of both walks.  label[m]: how a reason names member m; own[g]: the end of group g's own functions and
    // PF, the files aerMax reports
    std::map<std::string, uint32_t> portRecord;
    std::vector<std::string> label;
    std::vector<uint32_t> own;
    auto read = [&](const std::string &base, const std::string &entry, const std::string &fn) {  // the new record's index
        for (const char *name : {"aer_dev_fatal", "aer_dev_nonfatal"}) {
            std::string s;
            aerReads++;
            if (!readAerFile || !readAerFile(base, entry, name, s)) s.clear();
            if (s.size() > KXPU_AER_FILE_MAX + 1) s.resize(KXPU_AER_FILE_MAX + 1);
            off.push_back(text.size());
            len.push_back((uint32_t)s.size());
            text += s;
        }
        who.push_back(fn);
        return (uint32_t)(who.size() - 1);
    };
    auto addPorts = [&](const std::vector<std::pair<std::string, std::string>> &ports) {  // empty without aerPortHealth
        label.resize(members.size());
        own.push_back((uint32_t)members.size());
        for (const auto &pa : ports) {
            auto it = portRecord.find(pa.first);
            if (it == portRecord.end()) it = portRecord.emplace(pa.first, read(basePath, pa.first, pa.first)).first;
            members.push_back(it->second);
            label.push_back(pa.first + " (PCIe port above " + pa.second + ")");
        }
    };
    for (size_t g = 0; g < iommuMap.size(); g++) {
        for (const NvidiaGpuDevice &d : iommuMap[g].second) members.push_back(read(basePath, d.addr, d.addr));
        const std::string &pf = iommuState[g].pf;  // set only under vfVgpuHealth or sriovPfAware
        if (!pf.empty()) {
            auto it = pfRecord.find(pf);
            if (it == pfRecord.end()) it = pfRecord.emplace(pf, read(basePath, pf, pf)).first;
            members.push_back(it->second);
        }
        addPorts(iommuState[g].aerPorts);
        goff.push_back((uint32_t)members.size());
    }
    for (size_t g = 0; g < mdevMap.size(); g++) {
        for (const MdevDevice &m : mdevMap[g].second) members.push_back(read(mdevBasePath, m.uuid + "/..", m.parent));
        const std::string &pf = mdevState[g].pf;  // set only under vgpuSriovAware
        if (!pf.empty()) {
            auto it = pfRecord.find(pf);
            if (it == pfRecord.end()) it = pfRecord.emplace(pf, read(basePath, pf, pf)).first;
            members.push_back(it->second);
        }
        addPorts(mdevState[g].aerPorts);
        goff.push_back((uint32_t)members.size());
    }
    const size_t n = who.size(), G = goff.size() - 1;
    std::vector<uint64_t> totals(2 * n + 1);
    std::vector<uint8_t> bits(G + 1);
    const int32_t rc = kxpu_aer_health(ctx_, (const uint8_t *)text.data(), text.size(), off.data(), len.data(), n,
                                       aerFatalLimit, aerNonFatalLimit, goff.data(), members.data(), G, totals.data(),
                                       bits.data());
    if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_aer_health", rc);
    for (size_t g = 0; g < G; g++) {
        std::string why;  // the first member over a limit, fatal before non-fatal
        for (int k = 0; k < 2 && why.empty(); k++)
            for (uint32_t m = goff[g]; m < goff[g + 1] && why.empty(); m++) {
                const uint64_t c = totals[2 * members[m] + k], limit = k ? aerNonFatalLimit : aerFatalLimit;
                if (c != UINT64_MAX && c > limit)
                    why = (label[m].empty() ? who[members[m]] : label[m]) + " reported " + std::to_string(c) + (k ? " non-fatal" : " fatal") +
                          " uncorrectable PCIe errors (limit " + std::to_string(limit) + ")";
            }
        uint64_t most[2] = {KXPU_METRICS_NO_VALUE, KXPU_METRICS_NO_VALUE};  // the highest known count of each severity
        for (int k = 0; k < 2; k++)
            for (uint32_t m = goff[g]; m < own[g]; m++) {  // the group's own functions and PF: not its ports
                const uint64_t c = totals[2 * members[m] + k];
                if (c != UINT64_MAX && (most[k] == KXPU_METRICS_NO_VALUE || c > most[k])) most[k] = c;
            }
        auto &st = g < iommuState.size() ? iommuState[g].aerMax : mdevState[g - iommuState.size()].aerMax;
        if (g < iommuState.size()) set(iommuState[g], why, bits[g]);
        else set(mdevState[g - iommuState.size()], why, bits[g]);
        st[0] = most[0];
        st[1] = most[1];
    }
    return Error();
}

void Plugin::updateAerTaints(bool &passthroughMoved, bool &vgpuMoved) {
    passthroughMoved = vgpuMoved = false;
    if (!draTaints || !aerHealth) {
        aerTaint_.clear();
        return;
    }
    const int64_t t = now ? now() : (int64_t)time(nullptr);
    std::map<std::string, std::pair<uint8_t, int64_t>> next;
    auto visit = [&](const std::string &g, uint8_t bits) {  // whether group g's taint changed
        const uint8_t v = (bits & KXPU_AER_FATAL) ? KXPU_AER_FATAL : (bits & KXPU_AER_NONFATAL) ? KXPU_AER_NONFATAL : 0;
        auto it = aerTaint_.find(g);
        const uint8_t was = it == aerTaint_.end() ? 0 : it->second.first;
        if (v) next[g] = {v, was == v ? it->second.second : t};  // a new value gets a new time
        return was != v;
    };
    forPublished(iommuMap, iommuState, xpuClasses, [&](const std::string &g, const auto &s) { passthroughMoved |= visit(g, s.aerBits); });
    forPublishedVfVgpu(iommuMap, iommuState, xpuClasses, [&](const std::string &g, const auto &s) { passthroughMoved |= visit(g, s.aerBits); });
    forPublished(mdevMap, mdevState, vgpuClasses, [&](const std::string &g, const auto &s) { vgpuMoved |= visit(g, s.aerBits); });
    aerTaint_ = std::move(next);
}

Error Plugin::refreshAerHealth(std::vector<size_t> &changedPlugins, bool &passthroughMoved, bool &vgpuMoved) {
    std::unique_lock<std::shared_mutex> lock(mu_);
    changedPlugins.clear();
    passthroughMoved = vgpuMoved = false;
    if (!aerHealth) return Error();
    Error e = computeAer();
    if (e) return e;
    const std::map<std::string, size_t> iommuAt = positions(iommuMap), mdevAt = positions(mdevMap);
    auto aerOf = [](const std::string &id, const std::map<std::string, size_t> &at, const auto &state) {
        auto it = at.find(id);
        return it == at.end() ? std::string() : state[it->second].aer;
    };
    for (size_t k = 0; k < devicePlugins.size(); k++) {
        bool moved = false;
        for (Device &d : devicePlugins[k].devs) {
            const std::string reason = devicePlugins[k].vgpu ? aerOf(d.ID, mdevAt, mdevState) : aerOf(d.ID, iommuAt, iommuState);
            moved |= d.aer.empty() != reason.empty();  // ListAndWatch sends health, not the reason
            d.aer = reason;
        }
        if (moved) changedPlugins.push_back(k);
    }
    updateAerTaints(passthroughMoved, vgpuMoved);
    if (passthroughMoved) pci_.draGeneration++;
    if (vgpuMoved) mdev_.draGeneration++;
    return Error();
}

Error Plugin::refreshVfVgpuTypes(std::vector<size_t> &changedPlugins, bool &passthroughMoved, bool &typesMoved) {
    std::unique_lock<std::shared_mutex> lock(mu_);
    changedPlugins.clear();
    passthroughMoved = typesMoved = false;
    if (!vfVgpuHealth) return Error();
    // the groups that vfVgpu plugins serve, in plugin order, each once; one record and one one-member group per VF
    const std::map<std::string, size_t> at = positions(iommuMap);
    std::vector<size_t> groups;
    std::set<size_t> seen;
    for (const GenericDevicePlugin &dp : devicePlugins) {
        if (dp.vgpu || !xpuClasses[dp.xpuClass].vfVgpu) continue;
        for (const Device &d : dp.devs) {
            auto it = at.find(d.ID);
            if (it != at.end() && !iommuMap[it->second].second.empty() && seen.insert(it->second).second) groups.push_back(it->second);
        }
    }
    const size_t n = groups.size();
    kxpu_vfvgpurec zero;
    memset(&zero, 0, sizeof zero);
    std::vector<kxpu_vfvgpurec> recs(n, zero);
    std::vector<uint32_t> was(n), goff(n + 1, 0), members(n), typeNow(n + 1), first(n + 1);
    std::vector<uint8_t> status(n + 1);
    for (size_t k = 0; k < n; k++) {
        const NvidiaGpuDevice &vf = iommuMap[groups[k]].second.front();
        readCurrentType(*this, vf.addr, recs[k]);
        was[k] = vf.vgpuType;
        members[k] = (uint32_t)k;
        goff[k + 1] = (uint32_t)(k + 1);
    }
    if (n) {
        const int32_t rc = kxpu_vf_vgpu_drift(ctx_, recs.data(), was.data(), n, goff.data(), members.data(), n, typeNow.data(),
                                              status.data(), first.data());
        if (rc != KXPU_OK) return kxfail(ctx_, "kxpu_vf_vgpu_drift", rc);
    }
    for (GroupState<kxpu_dradev> &s : iommuState) s.drift.clear();
    for (size_t k = 0; k < n; k++) {
        if (first[k] == KXPU_VD_STEADY) continue;
        const uint32_t i = members[goff[k] + first[k]];
        const std::string &bdf = iommuMap[groups[k]].second.front().addr, wasText = " (was " + std::to_string(was[i]) + ")";
        iommuState[groups[k]].drift = status[i] == KXPU_VD_BAD ? bdf + " has an unreadable vGPU type" + wasText
                                                               : bdf + " now carries vGPU type " + std::to_string(typeNow[i]) + wasText;
        typesMoved |= status[i] == KXPU_VD_CHANGED;
    }
    for (size_t k = 0; k < devicePlugins.size(); k++) {
        if (devicePlugins[k].vgpu) continue;
        bool moved = false;
        for (Device &d : devicePlugins[k].devs) {
            auto it = at.find(d.ID);
            const std::string &reason = it == at.end() ? std::string() : iommuState[it->second].drift;
            moved |= d.drift.empty() != reason.empty();  // ListAndWatch sends health, not the reason
            d.drift = reason;
        }
        if (moved) changedPlugins.push_back(k);
    }
    if (!draTaints) return Error();
    const int64_t t = now ? now() : (int64_t)time(nullptr);
    std::map<std::string, int64_t> next;
    forPublishedVfVgpu(iommuMap, iommuState, xpuClasses, [&](const std::string &g, const GroupState<kxpu_dradev> &s) {
        auto it = driftTaint_.find(g);
        const bool had = it != driftTaint_.end(), has = !s.drift.empty();
        if (has) next[g] = had ? it->second : t;  // the time the drift was first seen, kept while it lasts
        passthroughMoved |= had != has;
    });
    driftTaint_ = std::move(next);
    if (passthroughMoved) pci_.draGeneration++;
    return Error();
}

Error Plugin::refreshDraHealth(bool &passthroughMoved, bool &vgpuMoved) {
    std::unique_lock<std::shared_mutex> lock(mu_);
    passthroughMoved = vgpuMoved = false;
    if (!draTaints) return Error();
    std::set<std::pair<bool, std::string>> unhealthy;  // (vgpu, group) that some plugin serving it has Unhealthy
    for (const GenericDevicePlugin &dp : devicePlugins)
        for (const Device &d : dp.devs)
            if (d.Health != kHealthy) unhealthy.insert({dp.vgpu, d.ID});
    const int64_t t = now ? now() : (int64_t)time(nullptr);
    std::map<std::string, int64_t> next;
    auto visit = [&](const std::string &g, bool vgpu) {  // whether group g's taint changed
        auto it = draTaintSince_.find(g);
        const bool was = it != draTaintSince_.end(), is = unhealthy.count({vgpu, g}) > 0;
        if (is) next[g] = was ? it->second : t;  // the time it turned unhealthy, kept while it stays so
        return was != is;
    };
    forPublished(iommuMap, iommuState, xpuClasses, [&](const std::string &g, const auto &) { passthroughMoved |= visit(g, false); });
    forPublishedVfVgpu(iommuMap, iommuState, xpuClasses, [&](const std::string &g, const auto &) { passthroughMoved |= visit(g, false); });
    forPublished(mdevMap, mdevState, vgpuClasses, [&](const std::string &g, const auto &) { vgpuMoved |= visit(g, true); });
    draTaintSince_ = std::move(next);
    if (passthroughMoved) pci_.draGeneration++;
    if (vgpuMoved) mdev_.draGeneration++;
    return Error();
}

Error Plugin::VgpuResourceSlices(size_t vgpuClass, std::vector<uint8_t> &out, std::vector<uint64_t> &sliceOff) {
    std::shared_lock<std::shared_mutex> lock(mu_);
    if (vgpuClass >= vgpuClasses.size() || vgpuClasses[vgpuClass].draDriver.empty())
        return fail("VgpuResourceSlices: vGPU class " + std::to_string(vgpuClass) + " has no DRA driver");
    std::vector<kxpu_dramdev> devs;
    std::vector<kxpu_dramdevpf> pfDevs;  // vgpuSriovAware: the same devices with their PFs
    std::vector<kxpu_dramdevpcie> pcieDevs;  // draVgpuPcie: the same devices with their PFs (vgpuSriovAware) and ports
    std::vector<std::string> groups;
    forPublished(mdevMap, mdevState, vgpuClasses, [&](const std::string &g, const GroupState<kxpu_dramdev> &s) {
        if (s.klass != vgpuClass) return;
        groups.push_back(g);
        if (!vgpuSriovAware && !draVgpuPcie) {
            devs.push_back(*s.dra);
            return;
        }
        kxpu_dramdevpf d;
        memset(&d, 0, sizeof d);
        d.dev = *s.dra;
        if (vgpuSriovAware) {
            memcpy(d.physfn, s.pf.data(), std::min(s.pf.size(), sizeof d.physfn));
            memcpy(d.physfn_device, s.pfDevice.data(), std::min(s.pfDevice.size(), sizeof d.physfn_device));
        }
        if (!s.pfProduct.empty()) {  // the GPU's model, not the VF's
            memset(d.dev.product, 0, sizeof d.dev.product);
            d.dev.product_len = (uint8_t)std::min(s.pfProduct.size(), sizeof d.dev.product);
            memcpy(d.dev.product, s.pfProduct.data(), d.dev.product_len);
        }
        if (!draVgpuPcie) {
            pfDevs.push_back(d);
            return;
        }
        kxpu_dramdevpcie q;
        memset(&q, 0, sizeof q);
        q.pf = d;
        q.root_port = s.rootPort;
        q.pcie_switch = s.pcieSwitch;
        pcieDevs.push_back(q);
    });
    if (draVgpuPcie) {
        const char *domain = draPcieDomain.c_str();
        auto fn = [domain](kxpu_ctx *ctx, const char *driver, const char *pool, const char *node, uint64_t generation,
                           const kxpu_dramdevpcie *v, size_t n, const kxpu_dra_taint *taints, size_t nt, const int64_t *since,
                           uint8_t *o, size_t cap, size_t *len, uint64_t *off, size_t *ns) {
            return kxpu_dra_slices_mdev_pcie(ctx, driver, pool, node, generation, domain, v, n, taints, nt, since, o, cap,
                                             len, off, ns);
        };
        return draSlices(fn, "kxpu_dra_slices_mdev_pcie", vgpuClasses[vgpuClass].draDriver, mdev_.draGeneration, pcieDevs,
                         groups, out, sliceOff);
    }
    if (vgpuSriovAware)
        return draSlices(kxpu_dra_slices_mdev_pf, "kxpu_dra_slices_mdev_pf", vgpuClasses[vgpuClass].draDriver,
                         mdev_.draGeneration, pfDevs, groups, out, sliceOff);
    return draSlices(kxpu_dra_slices_mdev_taints, "kxpu_dra_slices_mdev_taints", vgpuClasses[vgpuClass].draDriver,
                     mdev_.draGeneration, devs, groups, out, sliceOff);
}

Error Plugin::VfVgpuResourceSlices(size_t xpuClass, std::vector<uint8_t> &out, std::vector<uint64_t> &sliceOff) {
    std::shared_lock<std::shared_mutex> lock(mu_);
    if (xpuClass >= xpuClasses.size() || xpuClasses[xpuClass].vgpuDraDriver.empty())
        return fail("VfVgpuResourceSlices: class " + std::to_string(xpuClass) + " has no vGPU DRA driver");
    std::vector<kxpu_dravfvgpu> devs;
    std::vector<kxpu_dravfvgpupcie> pcieDevs;  // draVgpuPcie: the same devices with the ports of their groups
    std::vector<std::string> groups;
    forPublishedVfVgpu(iommuMap, iommuState, xpuClasses, [&](const std::string &g, const GroupState<kxpu_dradev> &s) {
        if (s.klass != xpuClass) return;
        groups.push_back(g);
        if (!draVgpuPcie) {
            devs.push_back(*s.vfVgpuDra);
            return;
        }
        kxpu_dravfvgpupcie q;
        memset(&q, 0, sizeof q);
        q.dev = *s.vfVgpuDra;
        q.root_port = s.rootPort;
        q.pcie_switch = s.pcieSwitch;
        pcieDevs.push_back(q);
    });
    if (draVgpuPcie) {
        const char *domain = draPcieDomain.c_str();
        auto fn = [domain](kxpu_ctx *ctx, const char *driver, const char *pool, const char *node, uint64_t generation,
                           const kxpu_dravfvgpupcie *v, size_t n, const kxpu_dra_taint *taints, size_t nt,
                           const int64_t *since, uint8_t *o, size_t cap, size_t *len, uint64_t *off, size_t *ns) {
            return kxpu_dra_slices_vf_vgpu_pcie(ctx, driver, pool, node, generation, domain, v, n, taints, nt, since, o, cap,
                                                len, off, ns);
        };
        return draSlices(fn, "kxpu_dra_slices_vf_vgpu_pcie", xpuClasses[xpuClass].vgpuDraDriver, pci_.draGeneration,
                         pcieDevs, groups, out, sliceOff, vfVgpuHealth);
    }
    return draSlices(kxpu_dra_slices_vf_vgpu, "kxpu_dra_slices_vf_vgpu", xpuClasses[xpuClass].vgpuDraDriver,
                     pci_.draGeneration, devs, groups, out, sliceOff, vfVgpuHealth);
}

Error Plugin::PrepareDraDevices(const std::string &driver, const std::string &pool, const std::vector<std::string> &deviceNames,
                                std::vector<std::vector<std::string>> &cdiIds) {
    std::vector<std::string> groups;
    {
        std::shared_lock<std::shared_mutex> lock(mu_);  // Allocate takes it again below
        size_t cls = xpuClasses.size(), vcls = vgpuClasses.size();
        for (size_t c = 0; c < xpuClasses.size(); c++)
            if (!driver.empty() && (xpuClasses[c].draDriver == driver || xpuClasses[c].vgpuDraDriver == driver)) cls = c;
        for (size_t c = 0; c < vgpuClasses.size(); c++)
            if (!driver.empty() && vgpuClasses[c].draDriver == driver) vcls = c;
        const bool vgpu = vcls < vgpuClasses.size();
        if (cls == xpuClasses.size() && !vgpu) return fail("PrepareDraDevices: unknown DRA driver " + driver);
        if (pool != nodeName) return fail("PrepareDraDevices: unknown pool " + pool + " of driver " + driver);
        for (const std::string &name : deviceNames) {
            const std::string g = name.compare(0, 4, "vfio") == 0 ? name.substr(4) : std::string();
            bool found;  // a group of the driver's class
            if (vgpu) {
                const GroupState<kxpu_dramdev> *s = stateOf(mdevMap, mdevState, g);
                found = s && s->klass == vcls;
            } else {
                const GroupState<kxpu_dradev> *s = stateOf(iommuMap, iommuState, g);
                found = s && s->klass == cls;
                if (found && !s->drift.empty())  // vfVgpuHealth: the profile the claim asked for is gone
                    return fail("PrepareDraDevices: device " + name + " no longer carries its published vGPU type: " + s->drift);
            }
            if (!found) return fail("PrepareDraDevices: unknown device " + name + " in pool " + pool);
            // refused even when the claim tolerates the taint: the device node is missing, so the VM cannot start
            if (draTaints && draTaintSince_.count(g))
                return fail("PrepareDraDevices: device " + name + " is tainted " + driver + kDraTaintKeyName + "=" +
                            kDraTaintValue + ":" + kDraTaintEffect + ": the VFIO device node of IOMMU group " + g +
                            " is missing");
            groups.push_back(g);
        }
    }
    cdiIds.clear();
    for (const std::string &g : groups) {
        ContainerAllocateResponse resp;
        Error e = Allocate({g}, resp);
        if (e) return e;
        cdiIds.push_back(resp.CDIDevices);
    }
    return Error();
}

Error Plugin::ListAndWatchBytes(const GenericDevicePlugin &dp, std::vector<uint8_t> &out) {
    std::shared_lock<std::shared_mutex> lock(mu_);
    std::vector<uint32_t> groups;
    std::vector<uint8_t> healthy;
    std::vector<uint64_t> masks;
    for (const Device &d : dp.devs) {
        groups.push_back((uint32_t)strtoul(d.ID.c_str(), nullptr, 10));
        healthy.push_back(sentHealthy(d));
        masks.push_back(d.numa);
    }
    // topologyAware: Device.topology from each device's mask (the HealthWatcher's re-sends come through here too)
    const char *what = topologyAware ? "kxpu_lw_encode_topo" : "kxpu_lw_encode";
    auto encode = [&](uint8_t *o, size_t cap, size_t *len) {
        return topologyAware ? kxpu_lw_encode_topo(ctx_, groups.data(), healthy.data(), masks.data(), groups.size(), o, cap, len)
                             : kxpu_lw_encode(ctx_, groups.data(), healthy.data(), groups.size(), o, cap, len);
    };
    size_t len = 0;
    int32_t rc = encode(nullptr, 0, &len);
    if (rc != KXPU_OK && rc != KXPU_E_NOSPACE) return kxfail(ctx_, what, rc);
    out.resize(len);
    if (len == 0) return Error();
    rc = encode(out.data(), len, &len);
    if (rc != KXPU_OK) return kxfail(ctx_, what, rc);
    return Error();
}

// The length MetricsText keeps of a label string: all of it up to KXPU_METRICS_STRING_MAX bytes (the kernel's limit),
// else the limit moved back to the start of a UTF-8 sequence that would be split there, so that the cut adds no U+FFFD.
size_t metricsCut(const uint8_t *s, size_t len) {
    const size_t max = KXPU_METRICS_STRING_MAX;
    if (len <= max) return len;
    size_t k = max;  // s[max] is the first byte left out; the nearest non-continuation byte at most three in front of it
    while (k > max - 3 && (s[k] & 0xC0u) == 0x80u) k--;
    const uint32_t c = s[k], need = c < 0xC2u ? 0u : c < 0xE0u ? 1u : c < 0xF0u ? 2u : c < 0xF5u ? 3u : 0u;
    return k < max && need && k + need >= max ? k : max;  // a lead whose sequence the limit would split
}

Error Plugin::MetricsText(std::vector<uint8_t> &out) {
    std::shared_lock<std::shared_mutex> lock(mu_);
    out.clear();
    std::string strings;
    std::vector<kxpu_metricdev> devs;
    std::vector<kxpu_metricreason> reasons;
    auto put = [&strings](const std::string &s, uint64_t &off, uint32_t &len) {
        off = strings.size();
        len = (uint32_t)metricsCut((const uint8_t *)s.data(), s.size());
        strings.append(s, 0, len);
    };
    // an upper bound of the document: every label byte at most three bytes once repaired or escaped, and at most 128
    // bytes of names, literals and decimals per sample; the headers within 512
    size_t bound = 512;
    const std::map<std::string, size_t> iommuAt = positions(iommuMap), mdevAt = positions(mdevMap);
    for (const GenericDevicePlugin &dp : devicePlugins) {
        kxpu_metricdev proto;
        memset(&proto, 0, sizeof proto);
        put(dp.resourceNamespace + "/" + dp.devpluginName, proto.resource_off, proto.resource_len);
        const std::map<std::string, size_t> &at = dp.vgpu ? mdevAt : iommuAt;
        for (const Device &d : dp.devs) {
            kxpu_metricdev m = proto;
            m.group = (uint32_t)strtoul(d.ID.c_str(), nullptr, 10);  // as ListAndWatchBytes writes Device.ID
            m.healthy = sentHealthy(d) ? 1u : 0u;
            m.aer_fatal = m.aer_nonfatal = KXPU_METRICS_NO_VALUE;
            m.reason_off = reasons.size();
            std::string address;
            uint32_t blockerKind = KXPU_MR_NOT_VIABLE;
            const std::string *sriov = nullptr, *reset = nullptr;
            auto it = at.find(d.ID);
            if (it != at.end() && dp.vgpu) {
                const GroupState<kxpu_dramdev> &s = mdevState[it->second];
                address = mdevMap[it->second].second.front().uuid;
                blockerKind = s.blockerKind;
                m.aer_fatal = s.aerMax[0];
                m.aer_nonfatal = s.aerMax[1];
            } else if (it != at.end()) {
                const GroupState<kxpu_dradev> &s = iommuState[it->second];
                address = iommuMap[it->second].second.front().addr;
                blockerKind = s.blockerKind;
                sriov = &s.sriov;
                reset = &s.reset;
                m.aer_fatal = s.aerMax[0];
                m.aer_nonfatal = s.aerMax[1];
            }
            put(address, m.address_off, m.address_len);
            size_t details = 0;
            auto reason = [&](uint32_t kind, const std::string &detail) {
                kxpu_metricreason r;
                memset(&r, 0, sizeof r);
                r.kind = kind;
                put(detail, r.detail_off, r.detail_len);
                reasons.push_back(r);
                details += detail.size();
            };
            // in kind order; sriov and reset are computed even when an earlier check holds the blocker, the cdev check only
            // without a viability blocker, so a reason never computed has no entry
            if (d.Health != kHealthy) reason(KXPU_MR_VFIO_DEVICE_MISSING, std::string());
            if (!d.blocker.empty()) reason(blockerKind, d.blocker);
            if (sriov && !sriov->empty() && (d.blocker.empty() || blockerKind < KXPU_MR_SRIOV)) reason(KXPU_MR_SRIOV, *sriov);
            if (reset && !reset->empty() && (d.blocker.empty() || blockerKind < KXPU_MR_RESET)) reason(KXPU_MR_RESET, *reset);
            if (!d.aer.empty()) reason(KXPU_MR_PCIE_AER, d.aer);
            if (!d.drift.empty()) reason(KXPU_MR_VGPU_TYPE_CHANGED, d.drift);
            m.reason_count = (uint32_t)(reasons.size() - m.reason_off);
            bound += (3 + m.reason_count) * (128 + 3 * (size_t)(m.resource_len + m.address_len)) + 3 * details;
            devs.push_back(m);
        }
    }
    if (!devs.empty()) {  // with no device there is nothing for the GPU to write
        out.resize(bound);
        size_t len = 0;
        const int32_t rc = kxpu_metrics_devices(ctx_, devs.data(), devs.size(), (const uint8_t *)strings.data(), strings.size(),
                                                reasons.data(), reasons.size(), out.data(), out.size(), &len);
        if (rc != KXPU_OK) {
            out.clear();
            return kxfail(ctx_, "kxpu_metrics_devices", rc);
        }
        out.resize(len);
    }
    auto line = [&out](const std::string &l) { out.insert(out.end(), l.begin(), l.end()); };
    line(KXPU_METRICS_READS_HEAD);
    const std::pair<const char *, uint64_t> reads[] = {{"aer_dev", aerReads.load(std::memory_order_relaxed)},
                                                       {"vfio-dev", cdevReads.load(std::memory_order_relaxed)},
                                                       {"sriov", sriovReads.load(std::memory_order_relaxed)},
                                                       {"reset", resetReads.load(std::memory_order_relaxed)},
                                                       {"nvidia", vfVgpuReads.load(std::memory_order_relaxed)}};
    for (const auto &r : reads) line(std::string("kata_xpu_sysfs_reads_total{file=\"") + r.first + "\"} " + std::to_string(r.second) + "\n");
    line(KXPU_METRICS_VALIDATIONS_HEAD);
    line("kata_xpu_allocate_validations_total{path=\"live\"} " + std::to_string(liveValidations.load(std::memory_order_relaxed)) + "\n");
    line("kata_xpu_allocate_validations_total{path=\"snapshot\"} " + std::to_string(snapshotValidations.load(std::memory_order_relaxed)) + "\n");
    return Error();
}

DevicePluginOptions Plugin::GetDevicePluginOptions() const {
    DevicePluginOptions o;  // PreStartRequired: false (generic_device_plugin.go:255)
    o.GetPreferredAllocationAvailable = topologyAware || pcieTopologyAware || vgpuPcieTopologyAware;
    return o;
}

Error Plugin::GetPreferredAllocation(const GenericDevicePlugin &dp, const std::vector<ContainerPreferredAllocationRequest> &requests,
                                     std::vector<ContainerPreferredAllocationResponse> &responses) {
    std::shared_lock<std::shared_mutex> lock(mu_);
    responses.clear();
    // the reference's empty response (generic_device_plugin.go:378-386)
    if (!GetDevicePluginOptions().GetPreferredAllocationAvailable) return Error();
    std::map<std::string, uint32_t> posOf;
    std::vector<uint64_t> numa(dp.devs.size());
    std::vector<uint32_t> node(dp.devs.size());
    for (size_t d = 0; d < dp.devs.size(); d++) {
        posOf.emplace(dp.devs[d].ID, (uint32_t)d);
        numa[d] = dp.devs[d].numa;
        node[d] = dp.devs[d].pcieNode;
    }
    std::vector<uint32_t> availOff{0}, mustOff{0}, avail, must, size;
    auto positions = [&](const std::vector<std::string> &ids, std::vector<uint32_t> &to) {
        for (const std::string &id : ids) {
            auto it = posOf.find(id);
            if (it == posOf.end()) return fail("invalid preferred allocation request: unknown device: " + id);
            to.push_back(it->second);
        }
        return Error();
    };
    for (const ContainerPreferredAllocationRequest &r : requests) {
        Error e = positions(r.AvailableDeviceIDs, avail);
        if (!e) e = positions(r.MustIncludeDeviceIDs, must);
        if (e) return e;
        if (r.AllocationSize < 0) return fail("invalid preferred allocation request: negative allocation size");
        availOff.push_back((uint32_t)avail.size());
        mustOff.push_back((uint32_t)must.size());
        size.push_back((uint32_t)r.AllocationSize);
    }
    size_t total = 0;
    for (uint32_t s : size) total += s;
    std::vector<uint32_t> out(total ? total : 1), outOff(requests.size() + 1);
    // one forest for all passthrough plugins of the PCI walk, one for all vGPU plugins of the mdev walk
    const bool pcie = dp.vgpu ? vgpuPcieTopologyAware : pcieTopologyAware;
    const std::vector<uint32_t> &fParent = dp.vgpu ? mdevPcieParent : pcieParent;
    const std::vector<uint8_t> &fDepth = dp.vgpu ? mdevPcieDepth : pcieDepth;
    int32_t rc = pcie ? kxpu_preferred_allocation_pcie(ctx_, numa.data(), node.data(), numa.size(), fParent.data(),
                                                       fDepth.data(), fParent.size(), availOff.data(), avail.data(),
                                                       mustOff.data(), must.data(), size.data(), requests.size(), out.data(),
                                                       outOff.data())
                      : kxpu_preferred_allocation(ctx_, numa.data(), numa.size(), availOff.data(), avail.data(), mustOff.data(),
                                                  must.data(), size.data(), requests.size(), out.data(), outOff.data());
    if (rc != KXPU_OK) return kxfail(ctx_, pcie ? "kxpu_preferred_allocation_pcie" : "kxpu_preferred_allocation", rc);
    for (size_t q = 0; q < requests.size(); q++) {
        ContainerPreferredAllocationResponse resp;
        for (uint32_t k = outOff[q]; k < outOff[q + 1]; k++) resp.DeviceIDs.push_back(dp.devs[out[k]].ID);
        responses.push_back(std::move(resp));
    }
    return Error();
}

// ---------------------------------------------------------------------------- health (row 3 of SURVEY 8(f))
HealthWatcher::HealthWatcher(GenericDevicePlugin &dp, bool watchCreates) : dp_(dp), watchCreates_(watchCreates) {}

HealthWatcher::~HealthWatcher() {
    if (fd_ >= 0) close(fd_);
}

// filepath.Join(path, dev.ID): one separator, no trailing one
static std::string joinPath(const std::string &dir, const std::string &name) {
    if (dir.empty()) return name;
    return dir.back() == '/' ? dir + name : dir + "/" + name;
}

std::vector<std::string> HealthWatcher::nodesOf(const std::string &id) const {
    auto it = dp_.nodes.find(id);
    return it == dp_.nodes.end() ? std::vector<std::string>{id} : it->second;
}

Error HealthWatcher::start() {
    fd_ = inotify_init1(IN_NONBLOCK | IN_CLOEXEC);  // fsnotify.NewWatcher (:396)
    if (fd_ < 0) return fail(std::string("Unable to create fsnotify watcher: ") + strerror(errno));
    // fsnotify's inotify backend adds every path with this mask; only the ops healthCheck looks at matter
    const uint32_t mask = IN_DELETE_SELF | IN_MOVE_SELF | IN_ATTRIB | IN_MODIFY;
    for (const Device &dev : dp_.devs) {  // :421-430
        for (const std::string &node : nodesOf(dev.ID)) {
            const std::string devicePath = joinPath(dp_.devicePath, node);
            int wd = inotify_add_watch(fd_, devicePath.c_str(), mask);
            if (wd < 0) return fail("Unable to add device path to fsnotify watcher: " + devicePath + ": " + strerror(errno));
            wdToId_[wd] = dev.ID;
            wdToNode_[wd] = node;
        }
    }
    if (watchCreates_) {
        dirWd_ = inotify_add_watch(fd_, dp_.devicePath.c_str(), IN_CREATE | IN_MOVED_TO);
        if (dirWd_ < 0) return fail("Unable to add device directory to fsnotify watcher: " + dp_.devicePath + ": " + strerror(errno));
    }
    return Error();
}

// follows the device list and, for cdev plugins, the node names: a watch whose (ID, node) left is dropped
Error HealthWatcher::resync() {
    if (fd_ < 0) return fail("health watcher not started");
    std::set<std::pair<std::string, std::string>> want;
    for (const Device &dev : dp_.devs)
        for (const std::string &node : nodesOf(dev.ID)) want.insert({dev.ID, node});
    std::set<std::pair<std::string, std::string>> have;
    for (auto it = wdToId_.begin(); it != wdToId_.end();) {
        const std::pair<std::string, std::string> key{it->second, wdToNode_[it->first]};
        if (!want.count(key)) {
            inotify_rm_watch(fd_, it->first);  // the IN_IGNORED that follows finds no entry
            wdToNode_.erase(it->first);
            it = wdToId_.erase(it);
        } else {
            have.insert(key);
            ++it;
        }
    }
    Error err;
    const uint32_t mask = IN_DELETE_SELF | IN_MOVE_SELF | IN_ATTRIB | IN_MODIFY;
    for (const auto &kv : want) {
        if (have.count(kv)) continue;
        const std::string devicePath = joinPath(dp_.devicePath, kv.second);
        int wd = inotify_add_watch(fd_, devicePath.c_str(), mask);
        if (wd < 0) {
            err = fail("Unable to add device path to fsnotify watcher: " + devicePath + ": " + strerror(errno));
            if (dp_.nodes.count(kv.first)) setHealth(kv.first, kUnhealthy);  // a cdev node that is not there
            continue;
        }
        wdToId_[wd] = kv.first;
        wdToNode_[wd] = kv.second;
    }
    return err;
}

// ListAndWatch's loops over dpi.devs (:230-234, :239-243): every dev with that ID
int HealthWatcher::setHealth(const std::string &id, const char *health) {
    int changed = 0;
    for (Device &d : dp_.devs)
        if (d.ID == id && d.Health != health) { d.Health = health; changed++; }
    return changed;
}

int HealthWatcher::poll(int timeout_ms) {
    if (fd_ < 0) return -1;
    struct pollfd pfd = {fd_, POLLIN, 0};
    int pr = ::poll(&pfd, 1, timeout_ms);
    if (pr < 0) return errno == EINTR ? 0 : -1;
    if (pr == 0) return 0;
    int changed = 0;
    alignas(struct inotify_event) char buf[16384];
    for (;;) {
        ssize_t n = read(fd_, buf, sizeof buf);
        if (n <= 0) break;  // EAGAIN: queue drained
        for (char *p = buf; p < buf + n;) {
            const struct inotify_event *ev = reinterpret_cast<const struct inotify_event *>(p);
            p += sizeof(struct inotify_event) + ev->len;
            events_++;
            if (ev->wd == dirWd_ && ev->len > 0) {
                // fsnotify.Create of devicePath/<name> (:441-443)
                const std::string name(ev->name);
                for (const Device &d : dp_.devs) {
                    const std::vector<std::string> nodes = nodesOf(d.ID);
                    if (std::find(nodes.begin(), nodes.end(), name) == nodes.end()) continue;
                    // the old watch died with the old inode: watch the new file like a restarted healthCheck would
                    int wd = inotify_add_watch(fd_, joinPath(dp_.devicePath, name).c_str(),
                                               IN_DELETE_SELF | IN_MOVE_SELF | IN_ATTRIB | IN_MODIFY);
                    if (wd >= 0) { wdToId_[wd] = d.ID; wdToNode_[wd] = name; }
                    bool all = true;  // a group is Healthy again only when every member's node is back
                    for (const std::string &n : nodes) all &= access(joinPath(dp_.devicePath, n).c_str(), F_OK) == 0;
                    if (all) changed += setHealth(d.ID, kHealthy);
                    break;
                }
                continue;
            }
            auto it = wdToId_.find(ev->wd);
            if (it == wdToId_.end()) continue;
            if (ev->mask & (IN_DELETE_SELF | IN_MOVE_SELF))  // fsnotify.Remove / fsnotify.Rename (:444-448)
                changed += setHealth(it->second, kUnhealthy);
            if (ev->mask & IN_IGNORED) { wdToNode_.erase(ev->wd); wdToId_.erase(it); }  // the kernel dropped the watch (file gone)
        }
    }
    return changed;
}

}  // namespace device_plugin

// ----------------------------------------------------------------------------------------
// C surface for the Python tests (tests/test_host*.py): drives the class above the way
// cmd/main.go drives the Go package.
// ----------------------------------------------------------------------------------------
using device_plugin::Plugin;

static void jstr(std::string &o, const std::string &s) {
    o += '"';
    for (char c : s) { if (c == '"' || c == '\\') o += '\\'; o += c; }
    o += '"';
}

static int copy_out(const std::string &s, char *out, size_t cap) {
    if (s.size() + 1 > cap) return -1;
    memcpy(out, s.c_str(), s.size() + 1);
    return (int)s.size();
}

extern "C" {

// CPU only: the raw gather of createIommuDeviceMap (no GPU involved)
int kxh_gather(const char *base_path, kxpu_devrec *out, size_t cap, size_t *n, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    std::vector<kxpu_devrec> recs;
    device_plugin::Error e = p.gatherRecords(recs);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_devrec));
    return 0;
}

// the batched / threaded variant of the same gather (SURVEY 8(f) row 2)
int kxh_gather_fast(const char *base_path, unsigned threads, kxpu_devrec *out, size_t cap, size_t *n, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    std::vector<kxpu_devrec> recs;
    device_plugin::Error e = p.gatherRecordsFast(recs, threads);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_devrec));
    return 0;
}

// "vendor,driver,namespace,kind,stem;..." -> class list; false on a malformed spec
static bool parseClasses(const char *spec, std::vector<device_plugin::XpuClass> &out) {
    out.clear();
    std::string all(spec), item;
    size_t pos = 0;
    while (pos <= all.size()) {
        size_t semi = all.find(';', pos);
        if (semi == std::string::npos) semi = all.size();
        item = all.substr(pos, semi - pos);
        pos = semi + 1;
        if (item.empty()) continue;
        std::vector<std::string> f;
        size_t a = 0;
        for (;;) {
            size_t c = item.find(',', a);
            f.push_back(item.substr(a, c == std::string::npos ? std::string::npos : c - a));
            if (c == std::string::npos) break;
            a = c + 1;
        }
        if (f.size() != 5 && !(f.size() == 6 && (f[5] == "cdev" || f[5] == "mdev-cdev"))) return false;
        out.push_back(device_plugin::XpuClass{f[0], f[1], f[2], f[3], f[4]});
        out.back().vfioCdev = f.size() == 6 && f[5] == "cdev";
        out.back().mdevCdev = f.size() == 6 && f[5] == "mdev-cdev";
    }
    return !out.empty();
}

// CPU only: the raw gather under a class list (fast = the batched / threaded variant)
int kxh_gather_classes(const char *base_path, const char *classes, int fast, unsigned threads, kxpu_devrec *out, size_t cap,
                       size_t *n, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    if (!parseClasses(classes, p.xpuClasses)) { copy_out("malformed class list", err, errcap); return -1; }
    std::vector<kxpu_devrec> recs;
    device_plugin::Error e = fast ? p.gatherRecordsFast(recs, threads) : p.gatherRecords(recs);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_devrec));
    return 0;
}

// CPU only: the raw gather under a class list ("...,cdev" marks a vfioCdev class) with the walk's cdev side array
// (-1 = none or not read) and the number of vfio-dev/ directories listed
int kxh_gather_cdev(const char *base_path, const char *classes, int fast, unsigned threads, kxpu_devrec *out, int64_t *cdevs,
                    size_t cap, size_t *n, uint64_t *reads, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    if (!parseClasses(classes, p.xpuClasses)) { copy_out("malformed class list", err, errcap); return -1; }
    std::vector<kxpu_devrec> recs;
    std::vector<int64_t> cd;
    device_plugin::Error e = fast ? p.gatherRecordsFast(recs, threads, nullptr, &cd) : p.gatherRecords(recs, nullptr, &cd);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    *reads = p.cdevReads;
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_devrec));
    for (size_t i = 0; i < recs.size(); i++) cdevs[i] = cd.empty() ? -1 : cd[i];
    return 0;
}

// CPU only: Plugin::checkVgpuClasses for these class lists
int kxh_check_vgpu_classes(const char *classes, const char *vgpu_classes, char *err, size_t errcap) {
    Plugin p(nullptr);
    if (!parseClasses(classes, p.xpuClasses) || !parseClasses(vgpu_classes, p.vgpuClasses)) {
        copy_out("malformed class list", err, errcap);
        return -1;
    }
    device_plugin::Error e = p.checkVgpuClasses();
    if (e) { copy_out(e.message, err, errcap); return -1; }
    return 0;
}

// a plugin's devicePath and its cdev nodes: {"path": "...", "nodes": {"<id>": ["vfio<N>", ...]}, "blockers": {"<id>": "..."}}
int kxh_plugin_nodes(void *h, int plugin_index, char *out, size_t cap) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return -1;
    const device_plugin::GenericDevicePlugin &dp = p->devicePlugins[(size_t)plugin_index];
    std::string o = "{\"path\":";
    jstr(o, dp.devicePath);
    o += ",\"nodes\":{";
    bool first = true;
    for (const auto &kv : dp.nodes) {
        if (!first) o += ',';
        first = false;
        jstr(o, kv.first);
        o += ":[";
        for (size_t i = 0; i < kv.second.size(); i++) { if (i) o += ','; jstr(o, kv.second[i]); }
        o += ']';
    }
    o += "},\"blockers\":{";
    first = true;
    for (const auto &d : dp.devs) {
        if (d.blocker.empty()) continue;
        if (!first) o += ',';
        first = false;
        jstr(o, d.ID); o += ':'; jstr(o, d.blocker);
    }
    return copy_out(o + "}}", out, cap);
}
uint64_t kxh_cdev_reads(void *h) { return ((Plugin *)h)->cdevReads; }

// the class list of a plugin (xpuClasses seam)
int kxh_set_classes(void *h, const char *classes) {
    return parseClasses(classes, ((Plugin *)h)->xpuClasses) ? 0 : -1;
}

void *kxh_new(kxpu_ctx *ctx, const char *base_path, const char *pciids_path, const char *cdi_dir) {
    Plugin *p = new Plugin(ctx);
    p->basePath = base_path;
    p->pciIdsFilePath = pciids_path;
    p->cdiConfigPath = cdi_dir;
    return p;
}
void kxh_free(void *h) { delete (Plugin *)h; }

// the vGPU classes of a plugin (vgpuClasses seam), same spec format; "" clears them
int kxh_set_vgpu_classes(void *h, const char *classes) {
    Plugin *p = (Plugin *)h;
    if (!classes[0]) { p->vgpuClasses.clear(); return 0; }
    return parseClasses(classes, p->vgpuClasses) ? 0 : -1;
}
void kxh_set_mdev_base(void *h, const char *path) { ((Plugin *)h)->mdevBasePath = path; }
// the device path a plugin's health watcher watches (tests point it at a fake /dev/vfio)
int kxh_set_device_path(void *h, int plugin_index, const char *path) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return -1;
    p->devicePlugins[(size_t)plugin_index].devicePath = path;
    return 0;
}

// CPU only: the raw mdev gather under a vGPU class list ("...,mdev-cdev" marks an mdevCdev class) with the walk's cdev
// side array (-1 = none or not read) and the number of vfio-dev/ directories listed
int kxh_gather_mdev_cdev(const char *mdev_base, const char *classes, kxpu_mdevrec *out, int64_t *cdevs, size_t cap, size_t *n,
                         uint64_t *reads, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.mdevBasePath = mdev_base;
    if (!parseClasses(classes, p.vgpuClasses)) { copy_out("malformed class list", err, errcap); return -1; }
    std::vector<kxpu_mdevrec> recs;
    device_plugin::MdevWalk w;
    device_plugin::Error e = p.gatherMdevRecords(recs, &w);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    *reads = p.cdevReads;
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_mdevrec));
    for (size_t i = 0; i < recs.size(); i++) cdevs[i] = w.cdevs.empty() ? -1 : w.cdevs[i];
    return 0;
}

// CPU only: the raw mdev gather under a vGPU class list
int kxh_gather_mdev(const char *mdev_base, const char *classes, kxpu_mdevrec *out, size_t cap, size_t *n, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.mdevBasePath = mdev_base;
    if (!parseClasses(classes, p.vgpuClasses)) { copy_out("malformed class list", err, errcap); return -1; }
    std::vector<kxpu_mdevrec> recs;
    device_plugin::Error e = p.gatherMdevRecords(recs);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_mdevrec));
    return 0;
}

static std::string dumpState(Plugin *p);

// InitiateDevicePlugin + a JSON dump of the resulting state
int kxh_init(void *h, const char *format, char *json, size_t cap) {
    Plugin *p = (Plugin *)h;
    device_plugin::Error e = p->createIommuDeviceMap();
    if (!e) e = p->createMdevMap();
    if (!e) e = p->generateCDISpec(p->iommuMap, format);
    if (!e) e = p->generateMdevCDISpec(format);
    if (!e) e = p->createDevicePlugins();
    if (e) { copy_out(e.message, json, cap); return -1; }
    return copy_out(dumpState(p) + "}", json, cap);
}

static void jsnap(std::string &o, const std::vector<kxpu_snaprec> &snap) {
    o += '[';
    for (size_t i = 0; i < snap.size(); i++) {
        if (i) o += ',';
        o += '['; jstr(o, std::string(snap[i].key, strnlen(snap[i].key, sizeof snap[i].key)));
        o += ',' + std::to_string(snap[i].iommu_group) + ',' + std::to_string(snap[i].klass) + ',' + std::to_string(snap[i].tag) +
             ',' + std::to_string(snap[i].index) + ']';
    }
    o += ']';
}

void kxh_set_sriov(void *h, int on) { ((Plugin *)h)->sriovAware = on != 0; }

// ---- resets between tenants (tests)
// on != 0: resetCheck; methods_csv != NULL replaces resetMethods ("" = none)
void kxh_set_reset(void *h, int on, const char *methods_csv) {
    Plugin *p = (Plugin *)h;
    p->resetCheck = on != 0;
    if (!methods_csv) return;
    p->resetMethods.clear();
    std::string cur;
    for (const char *c = methods_csv;; c++) {
        if (*c == ',' || *c == 0) {
            if (!cur.empty()) p->resetMethods.push_back(cur);
            cur.clear();
            if (*c == 0) break;
        } else {
            cur += *c;
        }
    }
}
uint64_t kxh_reset_reads(void *h) { return ((Plugin *)h)->resetReads; }

// CPU only: the raw PCI gather under a class list with resetCheck = on, then the reset reads (Plugin::readResets): the
// records, their paths and side records, and resetReads.  With on = 0 paths and rrs are zero-filled.
int kxh_gather_reset(const char *base_path, const char *classes, int on, int fast, unsigned threads, kxpu_devrec *out,
                     kxpu_pcipath *paths_out, kxpu_resetrec *rrs_out, size_t cap, size_t *n, uint64_t *reads, char *err,
                     size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    p.resetCheck = on != 0;
    if (!parseClasses(classes, p.xpuClasses)) { copy_out("malformed class list", err, errcap); return -1; }
    std::vector<kxpu_devrec> recs;
    std::vector<kxpu_pcipath> paths;
    std::vector<kxpu_resetrec> rrs;
    device_plugin::Error e = fast ? p.gatherRecordsFast(recs, threads, &paths) : p.gatherRecords(recs, &paths);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    p.readResets(recs, rrs);
    *n = recs.size();
    *reads = p.resetReads;
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_devrec));
    for (size_t i = 0; i < recs.size(); i++) {
        if (paths.size() > i) paths_out[i] = paths[i];
        else memset(&paths_out[i], 0, sizeof paths_out[i]);
        if (rrs.size() > i) rrs_out[i] = rrs[i];
        else memset(&rrs_out[i], 0, sizeof rrs_out[i]);
    }
    return 0;
}
uint64_t kxh_sriov_reads(void *h) { return ((Plugin *)h)->sriovReads; }

// "id=name;id=name" -> vgpuTypeNames; false for a malformed list
static bool parseTypeNames(const char *spec, std::map<uint32_t, std::string> &out) {
    out.clear();
    std::string all(spec ? spec : ""), item;
    size_t pos = 0;
    while (pos < all.size()) {
        size_t semi = all.find(';', pos);
        if (semi == std::string::npos) semi = all.size();
        item = all.substr(pos, semi - pos);
        pos = semi + 1;
        const size_t eq = item.find('=');
        if (eq == std::string::npos || eq == 0) return false;
        out[(uint32_t)strtoul(item.substr(0, eq).c_str(), nullptr, 10)] = item.substr(eq + 1);
    }
    return true;
}

// vfVgpu of class cls (vgpu != 0: of vGPU class cls, which InitiateDevicePlugin refuses) and its vgpuTypeNames
int kxh_set_vf_vgpu(void *h, int vgpu, int cls, int on, const char *names) {
    Plugin *p = (Plugin *)h;
    std::vector<device_plugin::XpuClass> &list = vgpu ? p->vgpuClasses : p->xpuClasses;
    if (cls < 0 || (size_t)cls >= list.size()) return -1;
    list[cls].vfVgpu = on != 0;
    return parseTypeNames(names, list[cls].vgpuTypeNames) ? 0 : -1;
}
uint64_t kxh_vf_vgpu_reads(void *h) { return ((Plugin *)h)->vfVgpuReads; }

// resourceNames of class cls (vgpu != 0: of vGPU class cls, which InitiateDevicePlugin refuses) from "id=name;id=name"
int kxh_set_resource_names(void *h, int vgpu, int cls, const char *spec) {
    Plugin *p = (Plugin *)h;
    std::vector<device_plugin::XpuClass> &list = vgpu ? p->vgpuClasses : p->xpuClasses;
    if (cls < 0 || (size_t)cls >= list.size()) return -1;
    list[cls].resourceNames.clear();
    std::string all(spec ? spec : "");
    for (size_t pos = 0; pos < all.size();) {
        size_t semi = all.find(';', pos);
        if (semi == std::string::npos) semi = all.size();
        const std::string item = all.substr(pos, semi - pos);
        pos = semi + 1;
        const size_t eq = item.find('=');
        if (eq == std::string::npos) return -1;
        list[cls].resourceNames[item.substr(0, eq)] = item.substr(eq + 1);
    }
    return 0;
}

// the learned (type ID, type key) pairs as {"id":"key",...}
int kxh_vgpu_learned(void *h, char *json, size_t cap) {
    std::string o = "{";
    for (const auto &kv : ((Plugin *)h)->learnedVgpuTypes()) {
        if (o.size() > 1) o += ',';
        jstr(o, std::to_string(kv.first));
        o += ':';
        jstr(o, kv.second);
    }
    return copy_out(o + "}", json, cap);
}

// CPU only: the raw PCI gather under a class list, classes whose bit is set in vf_mask serving vGPUs on VFs; the side
// records and the number of nvidia/ files read
int kxh_gather_vf_vgpu(const char *base_path, const char *classes, uint32_t vf_mask, kxpu_devrec *out, kxpu_vfvgpurec *vts,
                       size_t cap, size_t *n, uint64_t *reads, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    if (!parseClasses(classes, p.xpuClasses)) { copy_out("malformed class list", err, errcap); return -1; }
    for (size_t k = 0; k < p.xpuClasses.size() && k < 32; k++) p.xpuClasses[k].vfVgpu = (vf_mask >> k) & 1u;
    device_plugin::PciWalk w;
    device_plugin::Error e = p.gatherVfVgpu(w);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = w.recs.size();
    *reads = p.vfVgpuReads;
    if (w.recs.size() > cap) return -2;
    memcpy(out, w.recs.data(), w.recs.size() * sizeof(kxpu_devrec));
    for (size_t i = 0; i < w.recs.size(); i++) {
        if (w.vts.empty()) memset(&vts[i], 0, sizeof vts[i]);
        else vts[i] = w.vts[i];
    }
    return 0;
}

// CPU only: the raw PCI gather under a class list with sriovAware = on, its SR-IOV side records and sriovReads
int kxh_gather_sriov(const char *base_path, const char *classes, int on, int fast, unsigned threads, kxpu_devrec *out,
                     kxpu_sriovrec *srs, size_t cap, size_t *n, uint64_t *reads, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    p.sriovAware = on != 0;
    if (!parseClasses(classes, p.xpuClasses)) { copy_out("malformed class list", err, errcap); return -1; }
    std::vector<kxpu_devrec> recs;
    std::vector<kxpu_sriovrec> sr;
    device_plugin::Error e = fast ? p.gatherRecordsFast(recs, threads, nullptr, nullptr, &sr)
                                  : p.gatherRecords(recs, nullptr, nullptr, &sr);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    *reads = p.sriovReads;
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_devrec));
    for (size_t i = 0; i < recs.size(); i++) {
        if (sr.empty()) memset(&srs[i], 0, sizeof srs[i]);
        else srs[i] = sr[i];
    }
    return 0;
}

// the state kxh_init reports, without the closing brace
static std::string dumpState(Plugin *p) {
    std::string o = "{\"iommuMap\":[";
    bool first = true;
    for (const auto &kv : p->iommuMap) {
        if (!first) o += ',';
        first = false;
        o += '['; jstr(o, kv.first); o += ",[";
        for (size_t i = 0; i < kv.second.size(); i++) {
            if (i) o += ',';
            o += '['; jstr(o, kv.second[i].addr); o += ',' + std::to_string(kv.second[i].index) + ']';
        }
        o += "]]";
    }
    o += "],\"deviceMap\":[";
    first = true;
    for (const auto &kv : p->deviceMap) {
        if (!first) o += ',';
        first = false;
        o += '['; jstr(o, kv.first); o += ",[";
        for (size_t i = 0; i < kv.second.size(); i++) { if (i) o += ','; jstr(o, kv.second[i]); }
        o += "]]";
    }
    o += "],\"plugins\":[";
    first = true;
    for (const auto &dp : p->devicePlugins) {
        if (!first) o += ',';
        first = false;
        o += "{\"name\":"; jstr(o, dp.devpluginName);
        o += ",\"resource\":"; jstr(o, dp.resourceNamespace + "/" + dp.devpluginName);
        o += ",\"socket\":"; jstr(o, dp.socketPath);
        o += ",\"devs\":[";
        for (size_t i = 0; i < dp.devs.size(); i++) {
            if (i) o += ',';
            o += '['; jstr(o, dp.devs[i].ID); o += ','; jstr(o, dp.devs[i].Health); o += ']';
        }
        o += "],\"class\":" + std::to_string(dp.xpuClass) + ",\"vgpu\":" + (dp.vgpu ? "true" : "false") + "}";
    }
    o += "],\"cdiFile\":"; jstr(o, p->lastCdiFile);
    o += ",\"iommuClass\":[";
    for (size_t i = 0; i < p->iommuState.size(); i++) o += (i ? "," : "") + std::to_string(p->iommuState[i].klass);
    o += "],\"deviceClass\":[";
    for (size_t i = 0; i < p->deviceClass.size(); i++) o += (i ? "," : "") + std::to_string(p->deviceClass[i]);
    o += "],\"cdiFiles\":[";
    for (size_t i = 0; i < p->cdiFiles.size(); i++) { if (i) o += ','; jstr(o, p->cdiFiles[i]); }
    o += "],\"mdevMap\":[";
    for (size_t g = 0; g < p->mdevMap.size(); g++) {
        if (g) o += ',';
        o += '['; jstr(o, p->mdevMap[g].first); o += ",[";
        for (size_t i = 0; i < p->mdevMap[g].second.size(); i++) {
            const device_plugin::MdevDevice &m = p->mdevMap[g].second[i];
            if (i) o += ',';
            o += '['; jstr(o, m.uuid); o += ','; jstr(o, m.parent);
            o += ',' + std::to_string(m.index) + ',' + std::to_string(m.vgpuClass) + ']';
        }
        o += "]]";
    }
    o += "],\"mdevClass\":[";
    for (size_t i = 0; i < p->mdevState.size(); i++) o += (i ? "," : "") + std::to_string(p->mdevState[i].klass);
    o += "],\"typeMap\":[";
    for (size_t t = 0; t < p->typeMap.size(); t++) {
        if (t) o += ',';
        o += '['; jstr(o, p->typeMap[t].first); o += ",[";
        for (size_t i = 0; i < p->typeMap[t].second.size(); i++) { if (i) o += ','; jstr(o, p->typeMap[t].second[i]); }
        o += "]]";
    }
    o += "],\"typeClass\":[";
    for (size_t i = 0; i < p->typeClass.size(); i++) o += (i ? "," : "") + std::to_string(p->typeClass[i]);
    o += "],\"mdevCdiFiles\":[";
    for (size_t i = 0; i < p->mdevCdiFiles.size(); i++) { if (i) o += ','; jstr(o, p->mdevCdiFiles[i]); }
    o += "],\"pciSnapshot\":";
    jsnap(o, p->pciSnapshot());
    o += ",\"mdevSnapshot\":";
    jsnap(o, p->mdevSnapshot());
    o += ",\"pciNext\":" + std::to_string(p->pciNextIndex()) + ",\"mdevNext\":" + std::to_string(p->mdevNextIndex());
    return o;
}

// rediscover + kxh_init's state + the report
int kxh_rediscover(void *h, const char *format, char *json, size_t cap) {
    Plugin *p = (Plugin *)h;
    device_plugin::RediscoverReport r;
    device_plugin::Error e = p->rediscover(r, format);
    if (e) { copy_out(e.message, json, cap); return -1; }
    std::string o = dumpState(p) + ",\"report\":{\"changed\":[";
    for (size_t i = 0; i < r.changedPlugins.size(); i++) o += (i ? "," : "") + std::to_string(r.changedPlugins[i]);
    o += "],\"added\":[";
    for (size_t i = 0; i < r.addedPlugins.size(); i++) o += (i ? "," : "") + std::to_string(r.addedPlugins[i]);
    o += "],\"written\":[";
    for (size_t i = 0; i < r.cdiFilesWritten.size(); i++) { if (i) o += ','; jstr(o, r.cdiFilesWritten[i]); }
    o += "]";
    for (const auto &c : {std::make_pair("pci", &r.pci), std::make_pair("mdev", &r.mdev)}) {
        o += ",\"" + std::string(c.first) + "\":{\"n_kept\":" + std::to_string(c.second->n_kept) +
             ",\"n_new\":" + std::to_string(c.second->n_new) + ",\"n_changed\":" + std::to_string(c.second->n_changed) +
             ",\"n_retired\":" + std::to_string(c.second->n_retired) +
             ",\"next_index_out\":" + std::to_string(c.second->next_index_out) + "}";
    }
    o += "}}";
    return copy_out(o, json, cap);
}
int kxh_discovery_stale(void *h) { return ((Plugin *)h)->discoveryStale() ? 1 : 0; }
// the mdev generation through a seam (tests), like kxh_snapshot_enable's PCI one
void kxh_mdev_generation_seam(void *h, const uint64_t *generation) {
    ((Plugin *)h)->mdevGeneration = [generation](uint64_t &g) { g = *generation; return true; };
}
int kxh_health_resync(void *w, char *err, size_t errcap) {
    device_plugin::Error e = ((device_plugin::HealthWatcher *)w)->resync();
    if (e) { copy_out(e.message, err, errcap); return -1; }
    return 0;
}

// Allocate for one container request; ids = comma separated IOMMU group ids
int kxh_allocate(void *h, const char *ids_csv, char *json, size_t cap) {
    Plugin *p = (Plugin *)h;
    std::vector<std::string> ids;
    std::string cur;
    for (const char *c = ids_csv; *c; c++) { if (*c == ',') { ids.push_back(cur); cur.clear(); } else cur += *c; }
    if (!cur.empty() || (ids_csv[0] && ids_csv[strlen(ids_csv) - 1] == ',')) ids.push_back(cur);
    device_plugin::ContainerAllocateResponse resp;
    device_plugin::Error e = p->Allocate(ids, resp);
    if (e) { copy_out(e.message, json, cap); return -1; }
    std::string o = "{\"envs\":{";
    bool first = true;
    for (const auto &kv : resp.Envs) { if (!first) o += ','; first = false; jstr(o, kv.first); o += ':'; jstr(o, kv.second); }
    o += "},\"cdi_devices\":[";
    for (size_t i = 0; i < resp.CDIDevices.size(); i++) { if (i) o += ','; jstr(o, resp.CDIDevices[i]); }
    o += "]}";
    return copy_out(o, json, cap);
}

// ---- snapshot validation of Allocate (SURVEY 8(f) row 2): tests drive the generation through the seam
void kxh_snapshot_enable(void *h, const uint64_t *generation, const int *healthy) {
    Plugin *p = (Plugin *)h;
    p->snapshotValidation = true;
    if (generation) p->bindGeneration = [generation, healthy](uint64_t &g) { g = *generation; return !healthy || *healthy != 0; };
}
void kxh_validation_counts(void *h, uint64_t *live, uint64_t *snapshot) {
    Plugin *p = (Plugin *)h;
    *live = p->liveValidations;
    *snapshot = p->snapshotValidations;
}
// BindWatcher's uevent parser, message by message (CPU tests): returns the generation after the message
uint64_t kxh_uevent_feed(void **w, const char *msg, size_t len) {
    if (!*w) *w = new device_plugin::BindWatcher();
    device_plugin::BindWatcher *bw = (device_plugin::BindWatcher *)*w;
    if (msg) bw->feed(msg, len);
    return bw->generation();
}
// the mdev counter of the same watcher (kxh_uevent_feed creates it)
uint64_t kxh_uevent_mdev_generation(void *w) { return ((device_plugin::BindWatcher *)w)->mdevGeneration(); }
void kxh_uevent_free(void *w) { delete (device_plugin::BindWatcher *)w; }
// the rediscovery spec writer (CPU tests): 1 = written, 0 = the file already held these bytes, -1 = error
int kxh_write_spec_atomic(const char *path, const uint8_t *doc, size_t len) {
    bool written = false;
    device_plugin::Error e = device_plugin::writeSpecFileAtomicForTests(path, doc, len, written);
    if (e) return -1;
    return written ? 1 : 0;
}
// the real socket: 0 = opened (and healthy), < 0 = this box does not allow it
int kxh_uevent_socket_ok() {
    device_plugin::BindWatcher bw;
    return bw.start() ? -1 : (bw.healthy() ? 0 : -2);
}

// ---- health watcher (tests): a plugin can be added by hand so that no GPU is needed for the host logic
int kxh_add_plugin(void *h, const char *name, const char *device_path, const char *ids_csv) {
    Plugin *p = (Plugin *)h;
    device_plugin::GenericDevicePlugin dp;
    dp.devpluginName = name;
    dp.devicePath = device_path;
    dp.socketPath = std::string(device_plugin::kDevicePluginPath) + "kata-xpu-" + name + ".sock";
    std::string cur;
    for (const char *c = ids_csv;; c++) {
        if (*c == ',' || *c == 0) {
            if (!cur.empty()) dp.devs.push_back(device_plugin::Device{cur, device_plugin::kHealthy});
            cur.clear();
            if (*c == 0) break;
        } else {
            cur += *c;
        }
    }
    p->devicePlugins.push_back(std::move(dp));
    return (int)p->devicePlugins.size() - 1;
}

void *kxh_health_start(void *h, int plugin_index, int watch_creates, char *err, size_t errcap) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return nullptr;
    auto *w = new device_plugin::HealthWatcher(p->devicePlugins[(size_t)plugin_index], watch_creates != 0);
    device_plugin::Error e = w->start();
    if (e) { copy_out(e.message, err, errcap); delete w; return nullptr; }
    return w;
}
int kxh_health_poll(void *w, int timeout_ms) { return ((device_plugin::HealthWatcher *)w)->poll(timeout_ms); }
void kxh_health_stop(void *w) { delete (device_plugin::HealthWatcher *)w; }

// "id=Health,id=Health,..." of one plugin; a device of a group that is not viable shows "id=Health/<blocker>"
int kxh_devs(void *h, int plugin_index, char *out, size_t cap) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return -1;
    std::string o;
    for (const auto &d : p->devicePlugins[(size_t)plugin_index].devs) {
        if (!o.empty()) o += ',';
        o += d.ID + "=" + d.Health;
        if (!d.blocker.empty()) o += "/" + d.blocker;
    }
    return copy_out(o, out, cap);
}

int kxh_list_and_watch(void *h, int plugin_index, uint8_t *out, size_t cap) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return -1;
    std::vector<uint8_t> b;
    if (p->ListAndWatchBytes(p->devicePlugins[(size_t)plugin_index], b)) return -1;
    if (b.size() > cap) return -2;
    memcpy(out, b.data(), b.size());
    return (int)b.size();
}

// MetricsText into out (cap bytes); *len = its size.  0, -1 with the message in err, -2 when cap is too small
// metricsCut (CPU tests)
size_t kxh_metrics_cut(const char *s, size_t len) { return device_plugin::metricsCut((const uint8_t *)s, len); }

int kxh_metrics(void *h, uint8_t *out, size_t cap, size_t *len, char *err, size_t errcap) {
    std::vector<uint8_t> b;
    device_plugin::Error e = ((Plugin *)h)->MetricsText(b);
    if (e) {
        snprintf(err, errcap, "%s", e.message.c_str());
        return -1;
    }
    *len = b.size();
    if (b.size() > cap) return -2;
    memcpy(out, b.data(), b.size());
    return 0;
}

// ---- NUMA topology (tests)
void kxh_set_topology(void *h, int on) { ((Plugin *)h)->topologyAware = on != 0; }
void kxh_options(void *h, int *pre_start_required, int *preferred_allocation_available) {
    const device_plugin::DevicePluginOptions o = ((Plugin *)h)->GetDevicePluginOptions();
    *pre_start_required = o.PreStartRequired;
    *preferred_allocation_available = o.GetPreferredAllocationAvailable;
}

// counting_seam != 0: readNumaNode is replaced by a wrapper of the default read that counts its calls into *numa_reads
static void numaSeam(Plugin &p, int counting_seam, uint64_t *numa_reads) {
    if (!counting_seam) return;
    auto dflt = p.readNumaNode;
    p.readNumaNode = [dflt, numa_reads](const std::string &base, const std::string &entry, std::string &out) {
        (*numa_reads)++;
        return dflt(base, entry, out);
    };
}

// CPU only: the raw PCI gather with topologyAware = topo; fast = the batched / threaded variant
int kxh_gather_topo(const char *base_path, int topo, int fast, unsigned threads, int counting_seam, kxpu_devrec *out, size_t cap,
                    size_t *n, uint64_t *numa_reads, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    p.topologyAware = topo != 0;
    *numa_reads = 0;
    numaSeam(p, counting_seam, numa_reads);
    std::vector<kxpu_devrec> recs;
    device_plugin::Error e = fast ? p.gatherRecordsFast(recs, threads) : p.gatherRecords(recs);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_devrec));
    return 0;
}

// CPU only: the raw mdev gather under a vGPU class list with topologyAware = topo
int kxh_gather_mdev_topo(const char *mdev_base, const char *classes, int topo, int counting_seam, kxpu_mdevrec *out, size_t cap,
                         size_t *n, uint64_t *numa_reads, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.mdevBasePath = mdev_base;
    p.topologyAware = topo != 0;
    *numa_reads = 0;
    numaSeam(p, counting_seam, numa_reads);
    if (!parseClasses(classes, p.vgpuClasses)) { copy_out("malformed class list", err, errcap); return -1; }
    std::vector<kxpu_mdevrec> recs;
    device_plugin::Error e = p.gatherMdevRecords(recs);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_mdevrec));
    return 0;
}

// ---- PCIe topology (tests)
void kxh_set_pcie_topology(void *h, int on) { ((Plugin *)h)->pcieTopologyAware = on != 0; }
void kxh_set_vgpu_pcie_topology(void *h, int on) { ((Plugin *)h)->vgpuPcieTopologyAware = on != 0; }

// CPU only: the raw PCI gather with pcieTopologyAware = pcie; counting_seam != 0 wraps readPciPath in a counter of its
// calls (*path_reads), which also sends the fast gather down the walk
int kxh_gather_pcie(const char *base_path, int pcie, int fast, unsigned threads, int counting_seam, kxpu_devrec *out,
                    kxpu_pcipath *paths_out, size_t cap, size_t *n, size_t *n_paths, uint64_t *path_reads, char *err,
                    size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    p.pcieTopologyAware = pcie != 0;
    *path_reads = 0;
    if (counting_seam) {
        auto dflt = p.readPciPath;
        p.readPciPath = [dflt, path_reads](const std::string &base, const std::string &entry, std::string &target) {
            (*path_reads)++;
            return dflt(base, entry, target);
        };
    }
    std::vector<kxpu_devrec> recs;
    std::vector<kxpu_pcipath> paths;
    device_plugin::Error e = fast ? p.gatherRecordsFast(recs, threads, &paths) : p.gatherRecords(recs, &paths);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    *n_paths = paths.size();
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_devrec));
    memcpy(paths_out, paths.data(), paths.size() * sizeof(kxpu_pcipath));
    return 0;
}

// "id=node,..." of one plugin's devices (the PCIe node each Device carries)
int kxh_devs_pcie(void *h, int plugin_index, char *out, size_t cap) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return -1;
    std::string o;
    for (const auto &d : p->devicePlugins[(size_t)plugin_index].devs) {
        if (!o.empty()) o += ',';
        o += d.ID + "=" + std::to_string(d.pcieNode);
    }
    return copy_out(o, out, cap);
}

// GetPreferredAllocation for plugin plugin_index.  spec: container requests separated by ';', each
// "<available ids csv>|<must-include ids csv>|<size>".  json: [[ids of request 0], ...]
int kxh_preferred_allocation(void *h, int plugin_index, const char *spec, char *json, size_t cap) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return -1;
    auto split = [](const std::string &s, char sep) {
        std::vector<std::string> v;
        size_t a = 0;
        for (;;) {
            size_t c = s.find(sep, a);
            v.push_back(s.substr(a, c == std::string::npos ? std::string::npos : c - a));
            if (c == std::string::npos) break;
            a = c + 1;
        }
        return v;
    };
    std::vector<device_plugin::ContainerPreferredAllocationRequest> reqs;
    if (spec[0]) {
        for (const std::string &item : split(spec, ';')) {
            std::vector<std::string> f = split(item, '|');
            if (f.size() != 3) { copy_out("malformed request", json, cap); return -1; }
            device_plugin::ContainerPreferredAllocationRequest r;
            if (!f[0].empty()) r.AvailableDeviceIDs = split(f[0], ',');
            if (!f[1].empty()) r.MustIncludeDeviceIDs = split(f[1], ',');
            r.AllocationSize = atoi(f[2].c_str());
            reqs.push_back(std::move(r));
        }
    }
    std::vector<device_plugin::ContainerPreferredAllocationResponse> resps;
    device_plugin::Error e = p->GetPreferredAllocation(p->devicePlugins[(size_t)plugin_index], reqs, resps);
    if (e) { copy_out(e.message, json, cap); return -1; }
    std::string o = "[";
    for (size_t q = 0; q < resps.size(); q++) {
        if (q) o += ',';
        o += '[';
        for (size_t i = 0; i < resps[q].DeviceIDs.size(); i++) { if (i) o += ','; jstr(o, resps[q].DeviceIDs[i]); }
        o += ']';
    }
    o += ']';
    return copy_out(o, json, cap);
}

// "id=mask,..." of one plugin's devices (the NUMA mask each Device carries)
int kxh_devs_numa(void *h, int plugin_index, char *out, size_t cap) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return -1;
    std::string o;
    for (const auto &d : p->devicePlugins[(size_t)plugin_index].devs) {
        if (!o.empty()) o += ',';
        o += d.ID + "=" + std::to_string(d.numa);
    }
    return copy_out(o, out, cap);
}

// ---- IOMMU group viability (tests)
// on != 0: groupViability; drivers_csv != NULL replaces viabilityDrivers ("" = none)
void kxh_set_viability(void *h, int on, const char *drivers_csv) {
    Plugin *p = (Plugin *)h;
    p->groupViability = on != 0;
    if (!drivers_csv) return;
    p->viabilityDrivers.clear();
    std::string cur;
    for (const char *c = drivers_csv;; c++) {
        if (*c == ',' || *c == 0) {
            if (!cur.empty()) p->viabilityDrivers.push_back(cur);
            cur.clear();
            if (*c == 0) break;
        } else {
            cur += *c;
        }
    }
}

// CPU only: the raw PCI gather under a class list with groupViability = on (drivers_csv as kxh_set_viability); fast = the
// batched / threaded variant.  counting_seam != 0 wraps readLink in a counter of the `driver` and `iommu_group` reads of
// entries whose vendor no class has (*foreign_reads), which also sends the fast gather down the walk
int kxh_gather_viab(const char *base_path, const char *classes, int on, const char *drivers_csv, int fast, unsigned threads,
                    int counting_seam, kxpu_devrec *out, size_t cap, size_t *n, uint64_t *foreign_reads, char *err, size_t errcap) {
    Plugin p(nullptr);
    p.basePath = base_path;
    if (!parseClasses(classes, p.xpuClasses)) { copy_out("malformed class list", err, errcap); return -1; }
    kxh_set_viability(&p, on, drivers_csv);
    *foreign_reads = 0;
    if (counting_seam) {
        auto dflt = p.readLink;
        auto readID = p.readIDFromFile;
        const std::vector<device_plugin::XpuClass> classList = p.xpuClasses;
        p.readLink = [dflt, readID, classList, foreign_reads](const std::string &base, const std::string &addr,
                                                               const std::string &link, std::string &o) {
            std::string v;
            bool known = false;
            if (readID(base, addr, "vendor", v) && v.size() > 2) {
                std::string id = v.substr(2);
                while (!id.empty() && id.back() == '\n') id.pop_back();
                for (const auto &c : classList) known = known || c.vendor == id;
            }
            if (!known) (*foreign_reads)++;
            return dflt(base, addr, link, o);
        };
    }
    std::vector<kxpu_devrec> recs;
    device_plugin::Error e = fast ? p.gatherRecordsFast(recs, threads) : p.gatherRecords(recs);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    *n = recs.size();
    if (recs.size() > cap) return -2;
    memcpy(out, recs.data(), recs.size() * sizeof(kxpu_devrec));
    return 0;
}

// ---- DRA ResourceSlices (ABI v9)
// draDriver of every class from a comma separated list (position = class; "" = not published), and the node name
int kxh_set_dra(void *h, const char *drivers_csv, const char *node_name) {
    Plugin *p = (Plugin *)h;
    std::string all(drivers_csv);
    size_t c = 0, a = 0;
    for (;;) {
        const size_t comma = all.find(',', a);
        if (c >= p->xpuClasses.size()) return -1;
        p->xpuClasses[c++].draDriver = all.substr(a, comma == std::string::npos ? std::string::npos : comma - a);
        if (comma == std::string::npos) break;
        a = comma + 1;
    }
    p->nodeName = node_name;
    return 0;
}
// InitiateDevicePlugin (the configuration checks first); the error message into err
int kxh_initiate(void *h, char *err, size_t cap) {
    device_plugin::Error e = ((Plugin *)h)->InitiateDevicePlugin();
    if (e) { copy_out(e.message, err, cap); return -1; }
    return 0;
}
// ResourceSlices of one class: -1 with the message in out, -2 when out or offs is too small (*len / *n_slices hold the
// sizes), else 0
int kxh_resource_slices(void *h, int cls, uint8_t *out, size_t cap, size_t *len, uint64_t *offs, size_t offcap, size_t *n_slices) {
    std::vector<uint8_t> o;
    std::vector<uint64_t> so;
    device_plugin::Error e = ((Plugin *)h)->ResourceSlices((size_t)cls, o, so);
    if (e) { copy_out(e.message, (char *)out, cap); return -1; }
    *len = o.size();
    *n_slices = so.size() - 1;
    if (o.size() > cap || so.size() > offcap) return -2;
    memcpy(out, o.data(), o.size());
    memcpy(offs, so.data(), so.size() * sizeof(uint64_t));
    return 0;
}
uint64_t kxh_dra_generation(void *h) { return ((Plugin *)h)->draGeneration(); }
// counting seams on a plugin: every numa_node read and every entry-link read of its gathers (through the walk) is counted
void kxh_count_reads(void *h, uint64_t *numa_reads, uint64_t *path_reads) {
    Plugin *p = (Plugin *)h;
    auto dn = p->readNumaNode;
    p->readNumaNode = [dn, numa_reads](const std::string &base, const std::string &entry, std::string &out) {
        (*numa_reads)++;
        return dn(base, entry, out);
    };
    auto dp = p->readPciPath;
    p->readPciPath = [dp, path_reads](const std::string &base, const std::string &entry, std::string &target) {
        (*path_reads)++;
        return dp(base, entry, target);
    };
}
// PrepareDraDevices; names_csv = comma separated device names.  json: [[cdi names of device 0], ...] or the message
int kxh_prepare_dra(void *h, const char *driver, const char *pool, const char *names_csv, char *json, size_t cap) {
    std::vector<std::string> names;
    std::string all(names_csv);
    for (size_t a = 0; !all.empty();) {
        const size_t comma = all.find(',', a);
        names.push_back(all.substr(a, comma == std::string::npos ? std::string::npos : comma - a));
        if (comma == std::string::npos) break;
        a = comma + 1;
    }
    std::vector<std::vector<std::string>> ids;
    device_plugin::Error e = ((Plugin *)h)->PrepareDraDevices(driver, pool, names, ids);
    if (e) { copy_out(e.message, json, cap); return -1; }
    std::string o = "[";
    for (size_t i = 0; i < ids.size(); i++) {
        o += i ? ",[" : "[";
        for (size_t k = 0; k < ids[i].size(); k++) { if (k) o += ','; jstr(o, ids[i][k]); }
        o += ']';
    }
    return copy_out(o + "]", json, cap);
}

// ---- DRA ResourceSlices of vGPUs (ABI v10)
// draDriver of every vGPU class from a comma separated list (position = vGPU class; "" = not published), and the node name
int kxh_set_vgpu_dra(void *h, const char *drivers_csv, const char *node_name) {
    Plugin *p = (Plugin *)h;
    std::string all(drivers_csv);
    size_t c = 0, a = 0;
    for (;;) {
        const size_t comma = all.find(',', a);
        if (c >= p->vgpuClasses.size()) return -1;
        p->vgpuClasses[c++].draDriver = all.substr(a, comma == std::string::npos ? std::string::npos : comma - a);
        if (comma == std::string::npos) break;
        a = comma + 1;
    }
    p->nodeName = node_name;
    return 0;
}
// VgpuResourceSlices of one vGPU class, answered like kxh_resource_slices
int kxh_vgpu_resource_slices(void *h, int cls, uint8_t *out, size_t cap, size_t *len, uint64_t *offs, size_t offcap,
                             size_t *n_slices) {
    std::vector<uint8_t> o;
    std::vector<uint64_t> so;
    device_plugin::Error e = ((Plugin *)h)->VgpuResourceSlices((size_t)cls, o, so);
    if (e) { copy_out(e.message, (char *)out, cap); return -1; }
    *len = o.size();
    *n_slices = so.size() - 1;
    if (o.size() > cap || so.size() > offcap) return -2;
    memcpy(out, o.data(), o.size());
    memcpy(offs, so.data(), so.size() * sizeof(uint64_t));
    return 0;
}
uint64_t kxh_dra_vgpu_generation(void *h) { return ((Plugin *)h)->draVgpuGeneration(); }

// ---- DRA ResourceSlices of vGPUs on SR-IOV VFs (kxpu_dra_slices_vf_vgpu)
// vgpuDraDriver of passthrough class cls (vgpu: of vGPU class cls; "" = not published), and the node name
int kxh_set_vf_vgpu_dra(void *h, int vgpu, int cls, const char *driver, const char *node_name) {
    Plugin *p = (Plugin *)h;
    std::vector<device_plugin::XpuClass> &classes = vgpu ? p->vgpuClasses : p->xpuClasses;
    if (cls < 0 || (size_t)cls >= classes.size()) return -1;
    classes[cls].vgpuDraDriver = driver;
    p->nodeName = node_name;
    return 0;
}
// VfVgpuResourceSlices of one class, answered like kxh_resource_slices
int kxh_vf_vgpu_slices(void *h, int cls, uint8_t *out, size_t cap, size_t *len, uint64_t *offs, size_t offcap,
                       size_t *n_slices) {
    std::vector<uint8_t> o;
    std::vector<uint64_t> so;
    device_plugin::Error e = ((Plugin *)h)->VfVgpuResourceSlices((size_t)cls, o, so);
    if (e) { copy_out(e.message, (char *)out, cap); return -1; }
    *len = o.size();
    *n_slices = so.size() - 1;
    if (o.size() > cap || so.size() > offcap) return -2;
    memcpy(out, o.data(), o.size());
    memcpy(offs, so.data(), so.size() * sizeof(uint64_t));
    return 0;
}
// a counting seam on readIDFromFile: every read of the file `prop` (e.g. "../device") is counted
void kxh_count_id_reads(void *h, const char *prop, uint64_t *reads) {
    Plugin *p = (Plugin *)h;
    auto di = p->readIDFromFile;
    const std::string want(prop);
    p->readIDFromFile = [di, want, reads](const std::string &base, const std::string &addr, const std::string &pr, std::string &out) {
        if (pr == want) (*reads)++;
        return di(base, addr, pr, out);
    };
}

// ---- DRA device taints (ABI v11)
void kxh_set_dra_taints(void *h, int on) { ((Plugin *)h)->draTaints = on != 0; }
// the clock of refreshDraHealth reads *t (tests); NULL restores time(nullptr)
void kxh_set_clock(void *h, const int64_t *t) {
    Plugin *p = (Plugin *)h;
    if (t) p->now = [t]() { return *t; };
    else p->now = nullptr;
}
// ---- PCIe AER health (ABI v12)
void kxh_set_aer_health(void *h, int on, uint64_t fatal_limit, uint64_t nonfatal_limit) {
    Plugin *p = (Plugin *)h;
    p->aerHealth = on != 0;
    p->aerFatalLimit = fatal_limit;
    p->aerNonFatalLimit = nonfatal_limit;
}
uint64_t kxh_aer_reads(void *h) { return ((Plugin *)h)->aerReads; }

// ---- restart resume of CDI indices (ABI v13)
void kxh_set_resume(void *h, int on) { ((Plugin *)h)->resumeIndices = on != 0; }
// kxh_init's state of the plugin as it stands (after kxh_initiate), with the resume report
int kxh_state(void *h, char *json, size_t cap) {
    Plugin *p = (Plugin *)h;
    const device_plugin::ResumeReport &r = p->resumeReport();
    std::string o = dumpState(p) + ",\"resume\":{";
    for (const auto &c : {std::make_pair("pci", &r.pci), std::make_pair("mdev", &r.mdev)}) {
        const kxpu_reconcile_counts &k = c.second->counts;
        o += "\"" + std::string(c.first) + "\":{\"n_kept\":" + std::to_string(k.n_kept) + ",\"n_new\":" + std::to_string(k.n_new) +
             ",\"n_changed\":" + std::to_string(k.n_changed) + ",\"n_retired\":" + std::to_string(k.n_retired) +
             ",\"next_index_out\":" + std::to_string(k.next_index_out) + ",\"files\":[";
        for (size_t i = 0; i < c.second->filesRead.size(); i++) { if (i) o += ','; jstr(o, c.second->filesRead[i]); }
        o += "],\"fallback\":";
        jstr(o, c.second->fallback);
        o += ",\"typed\":[";
        size_t k2 = 0;
        for (size_t cls : c.second->typedClasses) o += (k2++ ? "," : "") + std::to_string(cls);
        o += "]},";
    }
    o += "\"stateRead\":" + std::string(r.stateRead ? "true" : "false") + ",\"statePci\":" + std::to_string(r.statePci) +
         ",\"stateMdev\":" + std::to_string(r.stateMdev) + ",\"written\":[";
    for (size_t i = 0; i < r.filesWritten.size(); i++) { if (i) o += ','; jstr(o, r.filesWritten[i]); }
    o += "]}}";
    return copy_out(o, json, cap);
}
// CPU only: the index state file's text for (pci, mdev), and its parse (1 = well formed)
int kxh_index_state_format(uint64_t pci, uint64_t mdev, char *out, size_t cap) {
    return copy_out(device_plugin::formatIndexState(pci, mdev), out, cap);
}
int kxh_index_state_parse(const char *text, size_t len, uint64_t *pci, uint64_t *mdev) {
    return device_plugin::parseIndexState(std::string(text, len), *pci, *mdev) ? 1 : 0;
}
// refreshAerHealth: changed[0 .. *n_changed) = the plugins whose ListAndWatch bytes changed (at most cap written),
// *moved as kxh_refresh_dra_health's; -1 with the message in err
int kxh_refresh_aer_health(void *h, size_t *changed, size_t cap, size_t *n_changed, int *moved, char *err, size_t errcap) {
    std::vector<size_t> c;
    bool pt = false, vg = false;
    device_plugin::Error e = ((Plugin *)h)->refreshAerHealth(c, pt, vg);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    for (size_t k = 0; k < c.size() && k < cap; k++) changed[k] = c[k];
    *n_changed = c.size();
    *moved = (pt ? 1 : 0) | (vg ? 2 : 0);
    return 0;
}
// "id=<aer reason>,..." of one plugin (an empty reason: within the limits)
int kxh_devs_aer(void *h, int plugin_index, char *out, size_t cap) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return -1;
    std::string o;
    for (const auto &d : p->devicePlugins[(size_t)plugin_index].devs) {
        if (!o.empty()) o += ',';
        o += d.ID + "=" + d.aer;
    }
    return copy_out(o, out, cap);
}

// ---- health of vGPUs on SR-IOV VFs (kxpu_vf_vgpu_drift)
void kxh_set_vf_vgpu_health(void *h, int on) { ((Plugin *)h)->vfVgpuHealth = on != 0; }
void kxh_set_vgpu_sriov(void *h, int on) { ((Plugin *)h)->vgpuSriovAware = on != 0; }
void kxh_set_sriov_pf(void *h, int on) { ((Plugin *)h)->sriovPfAware = on != 0; }
void kxh_set_aer_port_health(void *h, int on) { ((Plugin *)h)->aerPortHealth = on != 0; }
void kxh_set_dra_pcie_domain(void *h, const char *domain) { ((Plugin *)h)->draPcieDomain = domain ? domain : ""; }
void kxh_set_dra_vgpu_pcie(void *h, int on) { ((Plugin *)h)->draVgpuPcie = on != 0; }
uint64_t kxh_mdev_physfn_reads(void *h) { return ((Plugin *)h)->mdevPhysfnReads; }
// refreshVfVgpuTypes: changed as kxh_refresh_aer_health's; *moved = bit 0 passthroughMoved, bit 1 typesMoved
int kxh_refresh_vf_vgpu_types(void *h, size_t *changed, size_t cap, size_t *n_changed, int *moved, char *err, size_t errcap) {
    std::vector<size_t> c;
    bool pt = false, types = false;
    device_plugin::Error e = ((Plugin *)h)->refreshVfVgpuTypes(c, pt, types);
    if (e) { copy_out(e.message, err, errcap); return -1; }
    for (size_t k = 0; k < c.size() && k < cap; k++) changed[k] = c[k];
    *n_changed = c.size();
    *moved = (pt ? 1 : 0) | (types ? 2 : 0);
    return 0;
}
// "id=<drift reason>,..." of one plugin (an empty reason: the walk's type)
int kxh_devs_drift(void *h, int plugin_index, char *out, size_t cap) {
    Plugin *p = (Plugin *)h;
    if (plugin_index < 0 || (size_t)plugin_index >= p->devicePlugins.size()) return -1;
    std::string o;
    for (const auto &d : p->devicePlugins[(size_t)plugin_index].devs) {
        if (!o.empty()) o += ',';
        o += d.ID + "=" + d.drift;
    }
    return copy_out(o, out, cap);
}

// refreshDraHealth: *moved = bit 0 passthrough pools, bit 1 vGPU pools; -1 with the message in err
int kxh_refresh_dra_health(void *h, int *moved, char *err, size_t cap) {
    bool pt = false, vg = false;
    device_plugin::Error e = ((Plugin *)h)->refreshDraHealth(pt, vg);
    if (e) { copy_out(e.message, err, cap); return -1; }
    *moved = (pt ? 1 : 0) | (vg ? 2 : 0);
    return 0;
}

}  // extern "C"
