"""A minimal HDF5 reader written from the file format specification (version 0 superblock files), for the tests.

It reads what an -st=h5 file and simple libhdf5 files hold: a superblock v0 found at 0, 512, 1024, ... (a user block puts a
nonzero base address in front of every address), the root group's symbol table (a v1 group B-tree of any depth over
symbol-table nodes, names in a local heap), and datasets whose v1 object headers carry a dataspace, an IEEE float datatype
(4 or 8 bytes, either byte order) and a contiguous layout.  Messages it does not need are skipped; continuation messages are
followed.  Besides the data it records the tree's structure, so that tests can check it.
"""
import struct

import numpy as np

SIGNATURE = b"\x89HDF\r\n\x1a\n"
UNDEF = 0xFFFFFFFFFFFFFFFF


class H5Error(Exception):
    pass


class Node:
    """One group B-tree node as found in the file."""

    def __init__(self, addr, level, entries, left, right, keys, children):
        self.addr, self.level, self.entries, self.left, self.right = addr, level, entries, left, right
        self.keys, self.children = keys, children  # keys: names (str), children: addresses


class H5File:
    def __init__(self, path):
        with open(path, "rb") as f:
            self.buf = f.read()
        self.size = len(self.buf)
        self.base = self._find_superblock()
        self._superblock()
        self.nodes = []      # every group B-tree node, in visiting order
        self.snods = []      # (address, number of symbols, allocated entries) of every symbol-table node
        self.datasets = {}   # name -> (dtype, shape, absolute data address)
        self.names = []      # dataset names in B-tree order
        self._group(self.root_btree, self.root_heap)

    # -- raw access (addresses are relative to the base address) --
    def _at(self, addr, n):
        a = self.base + addr
        if addr == UNDEF or a + n > self.size:
            raise H5Error("address %#x + %d is outside the file" % (addr, n))
        return self.buf[a:a + n]

    def _u(self, addr, n):
        return int.from_bytes(self._at(addr, n), "little")

    def _find_superblock(self):
        off = 0
        while off + 8 <= self.size:
            if self.buf[off:off + 8] == SIGNATURE:
                return off
            off = 512 if off == 0 else off * 2
        raise H5Error("no HDF5 signature")

    def _superblock(self):
        b = self.buf[self.base:self.base + 96]
        if len(b) < 96 or b[8] != 0:
            raise H5Error("only superblock version 0 is read")
        self.offset_size, self.length_size = b[13], b[14]
        if (self.offset_size, self.length_size) != (8, 8):
            raise H5Error("only 8-byte offsets and lengths are read")
        self.leaf_k, self.node_k = struct.unpack_from("<HH", b, 16)
        base_addr, self.freespace, self.eof, self.driver = struct.unpack_from("<4Q", b, 24)
        if base_addr != self.base:
            raise H5Error("base address %#x, superblock at %#x" % (base_addr, self.base))
        name_off, self.root_header, cache_type = struct.unpack_from("<QQI", b, 56)
        hdr_btree, hdr_heap = self._symbol_table_message(self.root_header)
        if cache_type == 1:
            self.root_btree, self.root_heap = struct.unpack_from("<QQ", b, 80)
            if (self.root_btree, self.root_heap) != (hdr_btree, hdr_heap):
                raise H5Error("root entry scratch pad disagrees with the root group's symbol table message")
        else:
            self.root_btree, self.root_heap = hdr_btree, hdr_heap

    # -- object headers (version 1) --
    def messages(self, addr):
        """[(type, flags, bytes)] of the v1 object header at addr, continuation blocks included"""
        if self._u(addr, 1) != 1:
            raise H5Error("object header at %#x is not version 1" % addr)
        nmsgs = self._u(addr + 2, 2)
        size = self._u(addr + 8, 4)
        blocks = [(addr + 16, size)]
        out = []
        while blocks and len(out) < nmsgs:
            p, n = blocks.pop(0)
            end = p + n
            while p + 8 <= end and len(out) < nmsgs:
                mtype, msize, mflags = struct.unpack("<HHB", self._at(p, 5))
                data = self._at(p + 8, msize)
                if mtype == 0x10:  # continuation
                    blocks.append(struct.unpack_from("<QQ", data))
                out.append((mtype, mflags, data))
                p += 8 + msize
        return out

    def _symbol_table_message(self, addr):
        for t, _, d in self.messages(addr):
            if t == 0x11:
                return struct.unpack_from("<QQ", d)
        raise H5Error("object at %#x is not a group" % addr)

    # -- local heap --
    def _heap(self, addr):
        if self._at(addr, 4) != b"HEAP":
            raise H5Error("no local heap at %#x" % addr)
        size, free, data = struct.unpack_from("<QQQ", self._at(addr + 8, 24))
        seg = self._at(data, size)
        return seg, free, data

    @staticmethod
    def _name(seg, off):
        end = seg.index(b"\0", off)
        return seg[off:end].decode()

    # -- group B-tree and symbol-table nodes --
    def _group(self, btree, heap):
        seg, self.heap_free, self.heap_data = self._heap(heap)
        self.heap_addr = heap
        self.heap_size = len(seg)
        self._node(btree, seg, None)

    def _node(self, addr, seg, want_level):
        if self._at(addr, 4) != b"TREE":
            raise H5Error("no B-tree node at %#x" % addr)
        ntype, level, entries = struct.unpack("<BBH", self._at(addr + 4, 4))
        if ntype != 0:
            raise H5Error("not a group B-tree node at %#x" % addr)
        if want_level is not None and level != want_level:
            raise H5Error("child at %#x has level %d, expected %d" % (addr, level, want_level))
        left, right = struct.unpack("<QQ", self._at(addr + 8, 16))
        p = addr + 24
        keys, children = [], []
        for i in range(entries):
            keys.append(self._name(seg, self._u(p, 8)))
            children.append(self._u(p + 8, 8))
            p += 16
        keys.append(self._name(seg, self._u(p, 8)))
        self.nodes.append(Node(addr, level, entries, left, right, keys, children))
        for c in children:
            if level > 0:
                self._node(c, seg, level - 1)
            else:
                self._snod(c, seg)

    def _snod(self, addr, seg):
        if self._at(addr, 4) != b"SNOD":
            raise H5Error("no symbol-table node at %#x" % addr)
        nsym = self._u(addr + 6, 2)
        self.snods.append((addr, nsym))
        for i in range(nsym):
            e = addr + 8 + 40 * i
            name = self._name(seg, self._u(e, 8))
            header = self._u(e + 8, 8)
            self.names.append(name)
            self.datasets[name] = self._dataset(header)

    # -- datasets --
    def _dataset(self, addr):
        shape = dtype = data = None
        for t, _, d in self.messages(addr):
            if t == 0x01:  # dataspace v1 or v2
                ver, rank, flags = d[0], d[1], d[2]
                off = 8 if ver == 1 else 4
                shape = tuple(struct.unpack_from("<%dQ" % rank, d, off))
            elif t == 0x03:  # datatype
                cls, ver = d[0] & 0x0F, d[0] >> 4
                size = struct.unpack_from("<I", d, 4)[0]
                if cls != 1 or size not in (4, 8):
                    raise H5Error("only 4- and 8-byte floats are read")
                dtype = np.dtype((">" if d[1] & 1 else "<") + ("f4" if size == 4 else "f8"))
            elif t == 0x08:  # data layout
                ver = d[0]
                if ver == 3:
                    if d[1] != 1:
                        raise H5Error("only contiguous datasets are read")
                    data = struct.unpack_from("<QQ", d, 2)
                elif ver in (1, 2):
                    rank, cls = d[1], d[2]
                    if cls != 1:
                        raise H5Error("only contiguous datasets are read")
                    data = (struct.unpack_from("<Q", d, 8)[0], None)
                else:
                    raise H5Error("layout message version %d" % ver)
        if shape is None or dtype is None or data is None:
            raise H5Error("object at %#x is not a dataset this reader knows" % addr)
        return dtype, shape, data[0], data[1]

    def read(self, name):
        dtype, shape, addr, nbytes = self.datasets[name]
        n = int(np.prod(shape)) * dtype.itemsize
        if nbytes is not None and nbytes != n:
            raise H5Error("dataset %s: layout size %d, dataspace needs %d" % (name, nbytes, n))
        return np.frombuffer(self._at(addr, n), dtype).reshape(shape).astype(dtype.newbyteorder("="))

    def lookup(self, name):
        """The object header address of `name`, found as libhdf5 finds it: from the root node down, the child i whose keys
        bound the name as keys[i] < name <= keys[i + 1] (strcmp order), then the symbol-table node's entries.  None if absent."""
        seg, _, _ = self._heap(self.root_heap)
        want = name.encode()
        addr = self.root_btree
        while True:
            level, entries = self._u(addr + 5, 1), self._u(addr + 6, 2)
            keys = [self._name(seg, self._u(addr + 24 + 16 * i, 8)).encode() for i in range(entries + 1)]
            kids = [self._u(addr + 32 + 16 * i, 8) for i in range(entries)]
            hit = [i for i in range(entries) if keys[i] < want <= keys[i + 1]]
            if not hit:
                return None
            addr = kids[hit[0]]
            if level == 0:
                for i in range(self._u(addr + 6, 2)):
                    e = addr + 8 + 40 * i
                    if self._name(seg, self._u(e, 8)).encode() == want:
                        return self._u(e + 8, 8)
                return None

    def addresses(self):
        """every address the structure holds (absolute), for bounds checks"""
        out = [self.base + self.root_header, self.base + self.heap_addr, self.base + self.heap_data]
        out += [self.base + n.addr for n in self.nodes] + [self.base + a for a, _ in self.snods]
        out += [self.base + d[2] for d in self.datasets.values()]
        return out
