"""Minimal RIFF/WAVE reader and writer (PCM 16/24/32, IEEE float 32/64) on numpy.

The reference delegates file I/O to libsndfile (matchering/loader.py:35, saver.py:32), which is
not in this image; file I/O is outside the accelerated hot path (SURVEY.md section 8f)."""
from __future__ import annotations

import os
import struct

import numpy as np

_PCM, _FLOAT, _EXTENSIBLE = 1, 3, 0xFFFE


def read(path: str):
    """-> (float64 array (frames, channels), sample_rate).  Raises RuntimeError on a bad file."""
    with open(path, "rb") as f:
        data = f.read()
    if len(data) < 12 or data[:4] != b"RIFF" or data[8:12] != b"WAVE":
        raise RuntimeError("Format not recognised")
    pos, fmt, payload = 12, None, None
    while pos + 8 <= len(data):
        cid, size = data[pos:pos + 4], struct.unpack("<I", data[pos + 4:pos + 8])[0]
        body = data[pos + 8:pos + 8 + size]
        if cid == b"fmt ":
            fmt = body
        elif cid == b"data":
            payload = body
        pos += 8 + size + (size & 1)
    if fmt is None or payload is None or len(fmt) < 16:
        raise RuntimeError("Format not recognised")
    tag, channels, rate, _, _, bits = struct.unpack("<HHIIHH", fmt[:16])
    if tag == _EXTENSIBLE and len(fmt) >= 26:
        tag = struct.unpack("<H", fmt[24:26])[0]
    if channels < 1:
        raise RuntimeError("Format not recognised")
    if tag == _PCM and bits == 16:
        x = np.frombuffer(payload, dtype="<i2").astype(np.float64) / 32768.0
    elif tag == _PCM and bits == 24:
        raw = np.frombuffer(payload[: len(payload) // 3 * 3], dtype=np.uint8).reshape(-1, 3).astype(np.int32)
        v = raw[:, 0] | (raw[:, 1] << 8) | (raw[:, 2] << 16)
        v = np.where(v >= 1 << 23, v - (1 << 24), v)
        x = v.astype(np.float64) / 8388608.0
    elif tag == _PCM and bits == 32:
        x = np.frombuffer(payload, dtype="<i4").astype(np.float64) / 2147483648.0
    elif tag == _FLOAT and bits == 32:
        x = np.frombuffer(payload, dtype="<f4").astype(np.float64)
    elif tag == _FLOAT and bits == 64:
        x = np.frombuffer(payload, dtype="<f8").astype(np.float64)
    else:
        raise RuntimeError("unknown format")
    frames = len(x) // channels
    return np.ascontiguousarray(x[: frames * channels].reshape(frames, channels)), int(rate)


def write(path: str, array: np.ndarray, sample_rate: int, subtype: str) -> None:
    """Float samples in [-1, 1] -> WAV.  Integer subtypes scale by 2^(bits-1)-1, round to nearest
    (ties to even) and clip, which is libsndfile's float->int conversion."""
    a = np.asarray(array, dtype=np.float64)
    if a.ndim == 1:
        a = a[:, None]
    channels = a.shape[1]
    if subtype in ("PCM_16", "PCM_24", "PCM_32"):
        bits = int(subtype[4:])
        top = float((1 << (bits - 1)) - 1)
        q = np.clip(np.rint(a * top), -top - 1, top).astype(np.int64)
        if bits == 16:
            payload = q.astype("<i2").tobytes()
        elif bits == 32:
            payload = q.astype("<i4").tobytes()
        else:
            u = (q & 0xFFFFFF).astype(np.uint32).reshape(-1)
            payload = np.stack([u & 0xFF, (u >> 8) & 0xFF, (u >> 16) & 0xFF], axis=1).astype(np.uint8).tobytes()
        tag = _PCM
    elif subtype == "FLOAT":
        bits, tag, payload = 32, _FLOAT, a.astype("<f4").tobytes()
    elif subtype == "DOUBLE":
        bits, tag, payload = 64, _FLOAT, a.astype("<f8").tobytes()
    else:
        raise TypeError(f"WAV format does not have {subtype} subtype")
    block = channels * bits // 8
    fmt = struct.pack("<HHIIHH", tag, channels, int(sample_rate), int(sample_rate) * block, block, bits)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", len(payload)) + payload
    if len(payload) & 1:
        body += b"\x00"
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", len(body)) + body)


_IO_POOL = None
_IO_SLICE = 4 << 20


def _sliced_io(fd: int, view: memoryview, offset: int, write: bool) -> None:
    """pread / pwrite of a large buffer in 4 MB slices on a few threads (the calls release the GIL): the copy between
    the page cache and the (pinned) buffer is a single-threaded memcpy per call; eight of them in parallel read a
    track several times faster (writes of new files did not gain)."""
    global _IO_POOL
    n = len(view)
    if n <= _IO_SLICE:
        done = 0
        while done < n:
            k = os.pwrite(fd, view[done:], offset + done) if write else os.preadv(fd, [view[done:]], offset + done)
            if k <= 0:
                raise OSError("short read" if not write else "short write")
            done += k
        return
    if _IO_POOL is None:
        from concurrent.futures import ThreadPoolExecutor
        _IO_POOL = ThreadPoolExecutor(max_workers=8, thread_name_prefix="mgb-io")

    def one(lo: int) -> None:
        hi = min(n, lo + _IO_SLICE)
        while lo < hi:
            k = os.pwrite(fd, view[lo:hi], offset + lo) if write else os.preadv(fd, [view[lo:hi]], offset + lo)
            if k <= 0:
                raise OSError("short read" if not write else "short write")
            lo += k

    list(_IO_POOL.map(one, range(0, n, _IO_SLICE)))


def write_pcm(path: str, pcm: np.ndarray, sample_rate: int, bits: int, channels: int = 2) -> None:
    """Already-quantised samples (int16 (frames, ch) or packed 24-bit uint8 (frames, 3*ch)) -> WAV.  The
    samples go from the caller's buffer (pinned, when they come from the device) straight into the file."""
    pcm = np.ascontiguousarray(pcm)
    nbytes = pcm.nbytes
    block = channels * bits // 8
    fmt = struct.pack("<HHIIHH", _PCM, channels, int(sample_rate), int(sample_rate) * block, block, bits)
    head = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", nbytes)
    prefix = b"RIFF" + struct.pack("<I", len(head) + nbytes + (nbytes & 1)) + head
    with open(path, "wb", buffering=0) as f:
        f.write(prefix)
        f.write(memoryview(pcm).cast("B"))  # (parallel slices measured slower here: a new file's pages are allocated under one lock)
        if nbytes & 1:
            f.write(b"\x00")


def _pcm_layout(f):
    """Walk the RIFF chunks of an open file without reading the samples.
    -> (data offset, data bytes, sample_rate, channels, bits) or None when it is not 16/24-bit PCM WAV."""
    head = f.read(12)
    if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"WAVE":
        return None
    fmt, data_at, data_size = None, None, None
    pos = 12
    while True:
        f.seek(pos)
        hdr = f.read(8)
        if len(hdr) < 8:
            break
        cid, size = hdr[:4], struct.unpack("<I", hdr[4:8])[0]
        if cid == b"fmt ":
            fmt = f.read(size)
        elif cid == b"data":
            data_at, data_size = pos + 8, size
        pos += 8 + size + (size & 1)
    if fmt is None or data_at is None or len(fmt) < 16:
        return None
    tag, channels, rate, _, _, bits = struct.unpack("<HHIIHH", fmt[:16])
    if tag == _EXTENSIBLE and len(fmt) >= 26:
        tag = struct.unpack("<H", fmt[24:26])[0]
    if tag != _PCM or bits not in (16, 24) or channels < 1:
        return None
    return data_at, data_size, int(rate), int(channels), int(bits)


def read_pcm(path: str, allocate=None):
    """Raw 16- or 24-bit PCM of a WAV file without converting it on the host:
    -> (samples, sample_rate, channels, bits) with samples int16 (frames, ch) or packed 24-bit uint8
    (frames, 3*ch); None when the file is not 16/24-bit PCM WAV.  `allocate(shape, dtype)` supplies the
    buffer the samples are read into (pinned memory, so that the device can DMA from it); default numpy."""
    with open(path, "rb", buffering=0) as f:
        layout = _pcm_layout(f)
        if layout is None:
            return None
        data_at, data_size, rate, channels, bits = layout
        block = channels * bits // 8
        size = os.fstat(f.fileno()).st_size
        frames = max(0, min(data_size, size - data_at)) // block
        shape = (frames, channels if bits == 16 else 3 * channels)
        dtype = np.int16 if bits == 16 else np.uint8
        raw = allocate(shape, dtype) if allocate is not None else np.empty(shape, dtype=dtype)
        _sliced_io(f.fileno(), memoryview(raw).cast("B"), data_at, write=False)
    return raw, rate, channels, bits
