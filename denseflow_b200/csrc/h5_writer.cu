// h5_writer.cu — the -st=h5 flow file: H5Fcreate / H5LTmake_dataset_float / H5Fclose as the reference's USE_HDF5 build calls
// them (src/utils.cpp:27-41, src/common.cpp:120-150), written from the HDF5 file format specification without libhdf5.  Host
// code only.  This is the one translation unit that reads DFB_USE_HDF5: the "hdf5" build variant defines it and relinks the
// default objects with this one; without it the entry points refuse as the reference's default build does (:241).
//
// The file is what libhdf5 writes by default for a root group of contiguous float datasets:
//   superblock v0 (8-byte offsets and lengths, group leaf K 4, internal K 16, base address 0) whose root symbol-table entry
//   caches the group's B-tree and local heap (cache type 1); the root group's v1 object header with a symbol-table message;
//   v1 group B-tree nodes (32 children) over symbol-table nodes (SNOD, 8 entries), both at full capacity; one local heap of
//   the names; per dataset a v1 object header (dataspace, IEEE f32 LE datatype, fill value v2, contiguous layout v3).
// Payloads are appended as they arrive and the metadata follows them at close, so memory is O(datasets); nothing in the
// file depends on the time, so the same calls give the same bytes.
#include <cerrno>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

#include "../../include/denseflow_b200.h"
#include "common.cuh"

#ifdef DFB_USE_HDF5

#include <algorithm>
#include <unordered_set>
#include <vector>

namespace {

constexpr uint64_t kUndef = ~uint64_t(0);       // the undefined address
constexpr uint64_t kHeapFreeNull = 1;           // end of a local heap's free list (libhdf5's H5HL_FREE_NULL)
constexpr int kLeafK = 4, kNodeK = 16;          // superblock group K values: SNODs hold 2 * 4 names, nodes 2 * 16 children
constexpr int kSnodNames = 2 * kLeafK, kNodeChildren = 2 * kNodeK;
constexpr uint64_t kSuperblockBytes = 96, kEntryBytes = 40;
constexpr uint64_t kSnodBytes = 8 + kSnodNames * kEntryBytes;                                // 328
constexpr uint64_t kNodeBytes = 24 + (uint64_t)(kNodeChildren + 1) * 8 + kNodeChildren * 8;  // 544
constexpr uint64_t kHeapHeaderBytes = 32;
constexpr uint64_t kRootHeaderBytes = 16 + 8 + 16;
constexpr uint64_t kDatasetHeaderBytes = 16 + (8 + 24) + (8 + 24) + (8 + 8) + (8 + 24);      // 128

uint64_t round8(uint64_t v) { return (v + 7) & ~uint64_t(7); }

// little-endian encoder of one metadata block
struct Bytes {
    std::vector<uint8_t> b;
    void u8(unsigned v) { b.push_back((uint8_t)v); }
    void u16(unsigned v) { le(v, 2); }
    void u32(uint64_t v) { le(v, 4); }
    void u64(uint64_t v) { le(v, 8); }
    void raw(const void *p, size_t n) { b.insert(b.end(), (const uint8_t *)p, (const uint8_t *)p + n); }
    void zeros(size_t n) { b.insert(b.end(), n, 0); }
    void pad_to(size_t n) { zeros(n - b.size()); }
    void le(uint64_t v, int n) {
        for (int i = 0; i < n; ++i) b.push_back((uint8_t)(v >> (8 * i)));
    }
    // a v1 object header message: type, data size (a multiple of 8), flags
    void msg(unsigned type, unsigned size, unsigned flags) {
        u16(type);
        u16(size);
        u8(flags);
        zeros(3);
    }
};

struct Dataset {
    std::string name;
    uint64_t rows, cols, addr, heap_off;
};

}  // namespace

struct dfb_h5_file {
    FILE *fp = nullptr;
    uint64_t eof = 0;  // bytes written so far
    std::vector<Dataset> ds;
    std::unordered_set<std::string> names;
    std::string error;  // the first failed write
};

namespace {

int fail_file(dfb_h5_file *f, int code, const std::string &msg) {
    if (f && f->error.empty()) f->error = msg;
    return dfb::fail_unbound(code, msg);
}

bool put(dfb_h5_file *f, const void *p, size_t n) {
    if (std::fwrite(p, 1, n, f->fp) != n) return false;
    f->eof += n;
    return true;
}

// One v1 object header: version 1, `n` messages, reference count 1, `size` bytes of messages after the 16-byte prefix.
void object_header(Bytes &o, unsigned n, uint64_t size) {
    o.u8(1);
    o.u8(0);
    o.u16(n);
    o.u32(1);
    o.u32(size);
    o.u32(0);  // messages start 8-byte aligned
}

void dataset_header(Bytes &o, const Dataset &d) {
    const size_t start = o.b.size();
    object_header(o, 4, kDatasetHeaderBytes - 16);
    o.msg(0x0001, 24, 0);  // dataspace v1: rank 2, no maximum dimensions
    o.u8(1);
    o.u8(2);
    o.u8(0);
    o.zeros(5);
    o.u64(d.rows);
    o.u64(d.cols);
    o.msg(0x0003, 24, 1);  // datatype v1, class 1 (floating point): IEEE f32 little-endian
    o.u8(0x11);
    o.u8(0x20);  // byte order LE, no padding, implied mantissa MSB
    o.u8(31);    // sign bit
    o.u8(0);
    o.u32(4);
    o.u16(0);   // bit offset
    o.u16(32);  // precision
    o.u8(23);   // exponent location, size
    o.u8(8);
    o.u8(0);  // mantissa location, size
    o.u8(23);
    o.u32(127);  // exponent bias
    o.zeros(4);
    o.msg(0x0005, 8, 1);  // fill value v2: late allocation, fill time "if set", no fill value defined
    o.u8(2);
    o.u8(2);
    o.u8(2);
    o.u8(0);
    o.zeros(4);
    o.msg(0x0008, 24, 0);  // data layout v3, contiguous
    o.u8(3);
    o.u8(1);
    o.u64(d.addr);
    o.u64(d.rows * d.cols * 4);
    o.zeros(6);
    if (o.b.size() - start != kDatasetHeaderBytes) throw std::logic_error("h5: dataset header size");
}

// One node of the group's v1 B-tree, allocated at 2K children: keys[0..n] are heap offsets (key 0: the node's left bound, key i:
// the last name below child i - 1), children[0..n-1] addresses of SNODs (level 0) or nodes one level down.
struct Node {
    int level;
    uint64_t addr;
    std::vector<uint64_t> keys, children;
};

void node_bytes(Bytes &o, const Node &n, uint64_t left, uint64_t right) {
    const size_t start = o.b.size();
    o.raw("TREE", 4);
    o.u8(0);  // group node
    o.u8(n.level);
    o.u16((unsigned)n.children.size());
    o.u64(left);
    o.u64(right);
    for (size_t i = 0; i < n.children.size(); ++i) {
        o.u64(n.keys[i]);
        o.u64(n.children[i]);
    }
    o.u64(n.keys[n.children.size()]);
    o.zeros(kNodeBytes - (o.b.size() - start));
}

}  // namespace

extern "C" {

int dfb_h5_create(const char *path, dfb_h5_file **out) {
    if (!out) return dfb::fail_unbound(DFB_ERR_INVALID_ARG, "out is null");
    *out = nullptr;
    if (!path) return dfb::fail_unbound(DFB_ERR_INVALID_ARG, "path is null");
    dfb_h5_file *f = new dfb_h5_file();
    f->fp = std::fopen(path, "wb");
    if (!f->fp) {
        delete f;
        return dfb::fail_unbound(DFB_ERR_INVALID_ARG, std::string("cannot create ") + path + ": " + std::strerror(errno));
    }
    const uint8_t zero[kSuperblockBytes] = {};  // the superblock is written at close, when the root group's addresses are known
    if (!put(f, zero, sizeof(zero))) {
        std::fclose(f->fp);
        delete f;
        return dfb::fail_unbound(DFB_ERR_INVALID_ARG, std::string("cannot write ") + path);
    }
    *out = f;
    return DFB_OK;
}

int dfb_h5_write_float(dfb_h5_file *f, const char *name, int rows, int cols, const float *data) {
    if (!f) return dfb::fail_unbound(DFB_ERR_INVALID_ARG, "file is null");
    if (!name || !data) return dfb::fail_unbound(DFB_ERR_INVALID_ARG, "null name or data");
    if (rows <= 0 || cols <= 0) return dfb::fail_unbound(DFB_ERR_INVALID_ARG, "rows and cols must be positive");
    std::string n(name[0] == '/' ? name + 1 : name);  // H5LT names are paths from the root group
    if (n.empty() || n.find('/') != std::string::npos)
        return dfb::fail_unbound(DFB_ERR_INVALID_ARG, std::string("dataset name '") + name + "' is not a name in the root group");
    if (f->names.count(n)) return dfb::fail_unbound(DFB_ERR_INVALID_ARG, "dataset " + n + " already exists");
    const uint64_t bytes = (uint64_t)rows * (uint64_t)cols * 4;
    Dataset d{n, (uint64_t)rows, (uint64_t)cols, f->eof, 0};
    if (!put(f, data, bytes)) return fail_file(f, DFB_ERR_INVALID_ARG, "write of dataset " + n + " failed: " + std::strerror(errno));
    f->names.insert(n);
    f->ds.push_back(std::move(d));
    return DFB_OK;
}

int dfb_h5_close(dfb_h5_file *f) {
    if (!f) return dfb::fail_unbound(DFB_ERR_INVALID_ARG, "file is null");
    int rc = f->error.empty() ? DFB_OK : dfb::fail_unbound(DFB_ERR_INVALID_ARG, f->error);
    try {
        if (rc == DFB_OK) {
            const size_t N = f->ds.size();
            // local heap: offset 0 is the empty string, then every name NUL-terminated and padded to 8, in insertion order
            Bytes heap;
            heap.zeros(8);
            for (Dataset &d : f->ds) {
                d.heap_off = heap.b.size();
                heap.raw(d.name.c_str(), d.name.size() + 1);
                heap.pad_to(round8(heap.b.size()));
            }
            std::vector<size_t> order(N);
            for (size_t i = 0; i < N; ++i) order[i] = i;
            std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return std::strcmp(f->ds[a].name.c_str(), f->ds[b].name.c_str()) < 0; });

            // metadata layout after the payloads: dataset headers, root header, SNODs, B-tree nodes, heap header, heap data
            const uint64_t base = round8(f->eof);
            uint64_t at = base + N * kDatasetHeaderBytes;
            const uint64_t root_addr = at;
            at += kRootHeaderBytes;
            const size_t nsnod = (N + kSnodNames - 1) / kSnodNames;
            const uint64_t snod0 = at;
            at += nsnod * kSnodBytes;
            // the tree, bottom up: level 0 over the SNODs, each further level over the one below, until one node remains
            std::vector<std::vector<Node>> levels;
            std::vector<uint64_t> kids(nsnod), last(nsnod);  // children of the level being built and the last name below each
            for (size_t s = 0; s < nsnod; ++s) {
                kids[s] = snod0 + s * kSnodBytes;
                last[s] = f->ds[order[std::min(N, (s + 1) * kSnodNames) - 1]].heap_off;
            }
            do {
                std::vector<Node> lv;
                std::vector<uint64_t> nk, nl;
                const size_t nn = std::max<size_t>(1, (kids.size() + kNodeChildren - 1) / kNodeChildren);
                for (size_t i = 0; i < nn; ++i) {
                    Node n{(int)levels.size(), at, {}, {}};
                    at += kNodeBytes;
                    n.keys.push_back(i == 0 ? 0 : last[i * kNodeChildren - 1]);
                    for (size_t c = i * kNodeChildren; c < std::min(kids.size(), (i + 1) * kNodeChildren); ++c) {
                        n.children.push_back(kids[c]);
                        n.keys.push_back(last[c]);
                    }
                    nk.push_back(n.addr);
                    nl.push_back(n.keys.back());
                    lv.push_back(std::move(n));
                }
                levels.push_back(std::move(lv));
                kids.swap(nk);
                last.swap(nl);
            } while (kids.size() > 1);
            const uint64_t btree_root = kids[0];
            const uint64_t heap_addr = at;
            at += kHeapHeaderBytes;
            const uint64_t heap_data = at;
            at += heap.b.size();
            const uint64_t eof = at;

            Bytes m;
            m.pad_to(base - f->eof);
            for (const Dataset &d : f->ds) dataset_header(m, d);
            object_header(m, 1, kRootHeaderBytes - 16);
            m.msg(0x0011, 16, 0);  // symbol table message: B-tree, local heap
            m.u64(btree_root);
            m.u64(heap_addr);
            for (size_t s = 0; s < nsnod; ++s) {
                const size_t start = m.b.size();
                const size_t first = s * kSnodNames, n = std::min(N, first + kSnodNames) - first;
                m.raw("SNOD", 4);
                m.u8(1);
                m.u8(0);
                m.u16((unsigned)n);
                for (size_t k = 0; k < n; ++k) {  // entries: name, object header, cache type 0 (nothing cached)
                    const size_t i = order[first + k];
                    m.u64(f->ds[i].heap_off);
                    m.u64(base + i * kDatasetHeaderBytes);
                    m.zeros(24);
                }
                m.zeros(kSnodBytes - (m.b.size() - start));
            }
            for (const auto &lv : levels)
                for (size_t i = 0; i < lv.size(); ++i)
                    node_bytes(m, lv[i], i > 0 ? lv[i - 1].addr : kUndef, i + 1 < lv.size() ? lv[i + 1].addr : kUndef);
            m.raw("HEAP", 4);
            m.zeros(4);  // version 0
            m.u64(heap.b.size());
            m.u64(kHeapFreeNull);  // no free space
            m.u64(heap_data);
            m.raw(heap.b.data(), heap.b.size());
            if (f->eof + m.b.size() != eof) throw std::logic_error("h5: metadata layout");

            Bytes sb;
            sb.raw("\x89HDF\r\n\x1a\n", 8);
            sb.u8(0);  // superblock, free-space, root group entry, reserved, shared header versions
            sb.u8(0);
            sb.u8(0);
            sb.u8(0);
            sb.u8(0);
            sb.u8(8);  // sizes of offsets and lengths
            sb.u8(8);
            sb.u8(0);
            sb.u16(kLeafK);
            sb.u16(kNodeK);
            sb.u32(0);  // file consistency flags
            sb.u64(0);  // base address
            sb.u64(kUndef);  // free-space info
            sb.u64(eof);
            sb.u64(kUndef);  // driver info
            sb.u64(0);       // root entry: link name offset, object header, cache type 1 with the B-tree and heap addresses
            sb.u64(root_addr);
            sb.u32(1);
            sb.u32(0);
            sb.u64(btree_root);
            sb.u64(heap_addr);
            if (sb.b.size() != kSuperblockBytes) throw std::logic_error("h5: superblock size");

            if (!put(f, m.b.data(), m.b.size()) || std::fseek(f->fp, 0, SEEK_SET) != 0 || std::fwrite(sb.b.data(), 1, sb.b.size(), f->fp) != sb.b.size())
                rc = fail_file(f, DFB_ERR_INVALID_ARG, std::string("write of the file's metadata failed: ") + std::strerror(errno));
        }
    } catch (const std::exception &e) {
        rc = dfb::fail_unbound(DFB_ERR_INVALID_ARG, e.what());
    }
    if (std::fclose(f->fp) != 0 && rc == DFB_OK) rc = dfb::fail_unbound(DFB_ERR_INVALID_ARG, std::string("close failed: ") + std::strerror(errno));
    delete f;
    return rc;
}

}  // extern "C"

#else  // the reference's default build (USE_HDF5 OFF)

struct dfb_h5_file {};

namespace {
int refuse() { return dfb::fail_unbound(DFB_ERR_UNSUPPORTED, "HDF5 support is not enabled, pls recompile"); }
}  // namespace

extern "C" {
int dfb_h5_create(const char *, dfb_h5_file **out) {
    if (out) *out = nullptr;
    return refuse();
}
int dfb_h5_write_float(dfb_h5_file *, const char *, int, int, const float *) { return refuse(); }
int dfb_h5_close(dfb_h5_file *) { return refuse(); }
}  // extern "C"

#endif
