"""Index of a `torch.save` archive: where every tensor leaf's bytes lie in the file,
found without reading them.

The reader side of the format `fast_torch_save` writes (and `torch.save` itself): a
stored (uncompressed) zip whose records are `<archive>/data.pkl`, `byteorder`, ... and one
`<archive>/data/<key>` record per storage.  `index_file(path)` returns

  * `records`: the payload file offset and size of every `data/<key>` record, taken from
    the central directory (ZIP64 end records and extra fields included: `fast_torch_save`
    writes them past 4 GiB) and the local headers (payload = local header offset + 30 +
    name length + extra length);
  * `tree`: the unpickled object, with every tensor leaf replaced by a `TensorLeaf`
    (storage key, dtype, storage offset, shape, stride, file offset of the storage).

The pickle is read with torch's `weights_only` unpickler, so a file is exactly as safe to
index as it is to `torch.load` with torch's default; `persistent_load` hands it storages
on the meta device, so no payload byte is read.  Compressed records, a big-endian
`byteorder`, the legacy (non-zip) format and truncated archives raise ValueError naming
the file: the agent never writes any of them.
"""

from __future__ import annotations

import io
import os
import struct
from collections.abc import Mapping
from dataclasses import dataclass
from typing import Any, Dict, Tuple

import torch
from torch import _weights_only_unpickler

_EOCD = 0x06054B50
_EOCD64 = 0x06064B50
_LOC64 = 0x07064B50
_CDH = 0x02014B50
_LFH = 0x04034B50
_U16, _U32 = 0xFFFF, 0xFFFFFFFF


@dataclass(frozen=True)
class TensorLeaf:
    key: str                  # storage key: the record <archive>/data/<key>
    dtype: torch.dtype
    storage_offset: int       # in elements
    shape: Tuple[int, ...]
    stride: Tuple[int, ...]
    file_offset: int          # file offset of the storage's first byte
    record_bytes: int

    @property
    def element_size(self) -> int:
        return torch.empty((), dtype=self.dtype).element_size()

    @property
    def numel(self) -> int:
        n = 1
        for s in self.shape:
            n *= s
        return n

    def span(self) -> Tuple[int, int]:
        """(first byte, end) of the elements the view touches, relative to the storage."""
        es = self.element_size
        if self.numel == 0:
            return self.storage_offset * es, self.storage_offset * es
        last = self.storage_offset + sum((s - 1) * st for s, st in zip(self.shape, self.stride))
        return self.storage_offset * es, (last + 1) * es


@dataclass
class FileIndex:
    path: str
    size: int
    records: Dict[str, Tuple[int, int]]   # storage key -> (payload file offset, bytes)
    tree: Any


def _bad(path: str, why: str) -> ValueError:
    return ValueError(f"{path}: {why}")


def _pread(fd: int, n: int, off: int) -> bytes:
    out = bytearray()
    while len(out) < n:
        b = os.pread(fd, n - len(out), off + len(out))
        if not b:
            break
        out += b
    return bytes(out)


def _central_directory(path: str, fd: int, size: int):
    """[(name, method, compressed size, size, local header offset)] of the archive."""
    if _pread(fd, 4, 0) != b"PK\x03\x04":
        raise _bad(path, "not a zip archive (the legacy torch.save format, or not a "
                         "torch.save file); only the zip format can be restored from")
    tail_len = min(size, 22 + _U16)
    tail = _pread(fd, tail_len, size - tail_len)
    at = tail.rfind(struct.pack("<I", _EOCD))
    if at < 0 or len(tail) - at < 22:
        raise _bad(path, "no end of central directory record: the archive is truncated")
    eocd = size - tail_len + at
    (_, _, _, _, n, cd_size, cd_off, _) = struct.unpack("<IHHHHIIH", tail[at:at + 22])
    if eocd >= 20:
        loc = _pread(fd, 20, eocd - 20)
        if len(loc) == 20 and struct.unpack("<I", loc[:4])[0] == _LOC64:
            z_off = struct.unpack("<IIQI", loc)[2]
            rec = _pread(fd, 56, z_off)
            if len(rec) != 56 or struct.unpack("<I", rec[:4])[0] != _EOCD64:
                raise _bad(path, "bad ZIP64 end of central directory record")
            _, _, _, _, _, _, _, n, cd_size, cd_off = struct.unpack("<IQHHIIQQQQ", rec)
        elif n == _U16 or cd_size == _U32 or cd_off == _U32:
            raise _bad(path, "ZIP64 end of central directory locator missing")
    if cd_off + cd_size > size:
        raise _bad(path, "the central directory lies past the end of the file: truncated")
    cd = _pread(fd, cd_size, cd_off)
    out, p = [], 0
    for _ in range(n):
        if p + 46 > len(cd) or struct.unpack("<I", cd[p:p + 4])[0] != _CDH:
            raise _bad(path, "corrupt central directory")
        (_, _, _, _, method, _, _, _, csize, usize, nlen, elen, clen, _, _, _,
         lho) = struct.unpack("<IHHHHHHIIIHHHHHII", cd[p:p + 46])
        name = cd[p + 46:p + 46 + nlen].decode("utf-8")
        extra = cd[p + 46 + nlen:p + 46 + nlen + elen]
        q = 0
        while q + 4 <= len(extra):
            tag, ln = struct.unpack("<HH", extra[q:q + 4])
            if tag == 0x0001:  # ZIP64: the overflowing values, in this order
                vals = list(struct.unpack(f"<{ln // 8}Q", extra[q + 4:q + 4 + ln - ln % 8]))
                if usize == _U32 and vals:
                    usize = vals.pop(0)
                if csize == _U32 and vals:
                    csize = vals.pop(0)
                if lho == _U32 and vals:
                    lho = vals.pop(0)
            q += 4 + ln
        out.append((name, method, csize, usize, lho))
        p += 46 + nlen + elen + clen
    return out


def _payload_offset(path: str, fd: int, lho: int) -> int:
    lfh = _pread(fd, 30, lho)
    if len(lfh) != 30 or struct.unpack("<I", lfh[:4])[0] != _LFH:
        raise _bad(path, f"no local header at offset {lho}: the archive is truncated or corrupt")
    nlen, elen = struct.unpack("<HH", lfh[26:30])
    return lho + 30 + nlen + elen


def _walk_leaves(value, fn):
    if torch.is_tensor(value):
        return fn(value)
    if isinstance(value, Mapping):
        out = type(value)() if type(value) is not dict else {}
        try:
            for k, v in value.items():
                out[k] = _walk_leaves(v, fn)
        except TypeError:  # a Mapping that cannot be built empty
            out = {k: _walk_leaves(v, fn) for k, v in value.items()}
        return out
    if isinstance(value, list):
        return [_walk_leaves(v, fn) for v in value]
    if isinstance(value, tuple) and not hasattr(value, "_fields"):
        return tuple(_walk_leaves(v, fn) for v in value)
    return value


def index_file(path: str) -> FileIndex:
    """Index the torch.save archive at `path` (see the module docstring)."""
    path = os.fspath(path)
    fd = os.open(path, os.O_RDONLY)
    try:
        size = os.fstat(fd).st_size
        entries = _central_directory(path, fd, size)
        if not entries:
            raise _bad(path, "empty archive")
        prefix = entries[0][0].split("/", 1)[0]
        by_name = {}
        for name, method, csize, usize, lho in entries:
            if method != 0:
                raise _bad(path, f"record {name} is compressed (method {method}); only stored "
                                 "records can be restored from")
            off = _payload_offset(path, fd, lho)
            if off + usize > size:
                raise _bad(path, f"record {name} ends past the end of the file: truncated")
            by_name[name] = (off, usize)

        def record(name):
            if f"{prefix}/{name}" not in by_name:
                return None
            off, n = by_name[f"{prefix}/{name}"]
            return _pread(fd, n, off)

        order = record("byteorder")
        if order is not None and order != b"little":
            raise _bad(path, f"byteorder {order.decode(errors='replace')!r}: only "
                             "little-endian files can be restored from")
        pkl = record("data.pkl")
        if pkl is None:
            raise _bad(path, "no data.pkl record")
    finally:
        os.close(fd)
    data = f"{prefix}/data/"
    records = {n[len(data):]: v for n, v in by_name.items() if n.startswith(data)}

    keys: Dict[int, Tuple[str, int]] = {}

    def persistent_load(saved_id):
        typename, storage_type, key, _location, numel = saved_id
        if typename not in ("storage", b"storage"):
            raise _bad(path, f"unknown persistent id {typename!r}")
        key = key.decode() if isinstance(key, bytes) else str(key)
        dtype = torch.uint8 if storage_type is torch.UntypedStorage else storage_type.dtype
        nbytes = numel * torch._utils._element_size(dtype)
        if key not in records:
            raise _bad(path, f"the pickle references storage {key}, which has no record")
        if nbytes > records[key][1]:
            raise _bad(path, f"storage {key} needs {nbytes} bytes, its record holds "
                             f"{records[key][1]}")
        storage = torch.UntypedStorage(nbytes, device="meta")
        keys[storage._cdata] = (key, nbytes)
        return torch.storage.TypedStorage(wrap_storage=storage, dtype=dtype, _internal=True)

    unpickler = _weights_only_unpickler.Unpickler(io.BytesIO(pkl), encoding="utf-8")
    unpickler.persistent_load = persistent_load
    try:
        obj = unpickler.load()
    except _weights_only_unpickler.UnpicklingError as e:
        raise _weights_only_unpickler.UnpicklingError(
            f"{path}: refused by torch's weights_only unpickler: {e}") from e

    def leaf(t: torch.Tensor) -> TensorLeaf:
        got = keys.get(t.untyped_storage()._cdata)
        if got is None:
            raise _bad(path, "a tensor leaf does not come from a storage record")
        key, _ = got
        off, n = records[key]
        out = TensorLeaf(key=key, dtype=t.dtype, storage_offset=t.storage_offset(),
                         shape=tuple(t.shape), stride=tuple(t.stride()), file_offset=off,
                         record_bytes=n)
        lo, hi = out.span()
        if lo < 0 or hi > n:
            raise _bad(path, f"a view of storage {key} spans bytes [{lo}, {hi}) of a "
                             f"{n}-byte record")
        return out

    return FileIndex(path=path, size=size, records=records, tree=_walk_leaves(obj, leaf))
