"""Frame ingest for the batched detector (SURVEY.md §8f N4): raw frames from a pipe into pinned host memory.

The reference reads `width*height*3` bytes per frame from an ffmpeg `-f rawvideo -pix_fmt bgr24` pipe into a fresh
bytes object, wraps it in numpy, and the consumer copies it again before use (`frame_loop`, clearcam.py:401-421;
`process_frame` :446-447).  Here the bytes land once, in a page-locked slot the GPU can DMA from:

  * `FrameMailbox`   one camera's latest frame (the reference's `raw_frame[cam]` / `frame_num[cam]`), three pinned slots:
                     one being written, one published, one possibly still held by the consumer — no copy, no tearing
  * `PipeReader`     the `frame_loop` thread: fill the mailbox from a byte stream, count short reads and reopen the stream
                     after more than five in a row (clearcam.py:407-412)
  * `CameraBatch.step_mailboxes` (cameras.py) takes every camera's unseen frame straight from its mailbox
  * `VideoReader`    a recorded video: every frame in order (none dropped), in runs of consecutive frames for
                     `CameraBatch.step_video`, filled on a thread into two alternating pinned run buffers

Frames are bgr24 (`-pix_fmt bgr24`, H*W*3 bytes) or, with `FrameMailbox(h, w, pix_fmt="yuv420p")`, yuv420p
(`-pix_fmt yuv420p`, H*W*3/2 bytes: half the pipe, pinned-memory and PCIe bytes, and no swscale conversion on the host;
the GPU converts them, see clearcam_b200/pixfmt.py).

A Motion-JPEG camera (`ffmpeg ... -c:v copy -f mjpeg -`) is read without decoding on the host:

  * `MjpegSplitter`  cuts the stream of concatenated JPEG files into files by walking their marker segments
  * `default_tables` the DHT segments of the ITU-T T.81 Annex K tables that a frame's scan uses and does not define
                     (Motion-JPEG frames usually carry none; libjpeg-turbo substitutes exactly these)
  * `JpegMailbox`    the FrameMailbox of such a camera: each slot holds one whole JPEG file
  * `VideoReader(..., pix_fmt="mjpeg")` runs of JPEG files of a recorded video

Spawning ffmpeg (and HLS recording, clearcam.py:310-371) stays with the caller: `PipeReader` takes any callable that
returns a readable binary stream, e.g. `lambda: subprocess.Popen(cmd, stdout=subprocess.PIPE).stdout`."""
import queue
import threading
import time
from typing import Callable, Optional, Tuple

import numpy as np

import torch

from .pixfmt import BGR24, MJPEG, check_pix_fmt, yuv420p_rows

# ITU-T T.81 Annex K.3 Huffman tables: the 16 code counts (BITS), then the symbols (HUFFVAL).  Slot 0 is the luminance
# table, slot 1 the chrominance table, as libjpeg's std_huff_tables and ffmpeg's mjpeg2jpeg install them.
_ANNEX_K = {
    (0, 0): bytes.fromhex("00010501010101010100000000000000000102030405060708090a0b"),
    (0, 1): bytes.fromhex("00030101010101010101010000000000000102030405060708090a0b"),
    (1, 0): bytes.fromhex(
        "0002010303020403050504040000017d01020300041105122131410613516107227114328191a1082342b1c11552d1f024336272820"
        "90a161718191a25262728292a3435363738393a434445464748494a535455565758595a636465666768696a737475767778797a83848"
        "5868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e"
        "4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa"),
    (1, 1): bytes.fromhex(
        "00020102040403040705040400010277000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a1"
        "62434e125f11718191a262728292a35363738393a434445464748494a535455565758595a636465666768696a737475767778797a828"
        "38485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e"
        "3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa"),
}
# bytes the four inserted DHT segments can add to a frame
TABLE_ROOM = sum(4 + 1 + len(t) for t in _ANNEX_K.values())


def default_tables(data) -> Tuple[int, bytes]:
    """(offset, segments): the DHT segments to insert at `offset` of the JPEG file `data` (bytes-like or uint8 array) so
    that its first scan finds every Huffman table it uses.  One segment per DC or AC table of slot 0 or 1 that the scan
    references and no DHT before it defines, in the order libjpeg writes them (slot 0 DC, AC, then slot 1 DC, AC), each
    byte for byte the segment cv2.imencode writes for that table.  (0, b"") when nothing is missing, or when the file has
    no scan header to read; tables of slots 2 and 3 are never inserted (libjpeg has no default for them)."""
    a = np.frombuffer(data, np.uint8) if not isinstance(data, np.ndarray) else data
    n, pos, have = len(a), 2, set()
    if n < 4 or a[0] != 0xFF or a[1] != 0xD8:
        return 0, b""
    while pos + 4 <= n:
        if a[pos] != 0xFF:
            return 0, b""
        m = int(a[pos + 1])
        if m == 0xFF:
            pos += 1
            continue
        if m == 0x01 or 0xD0 <= m <= 0xD7:
            pos += 2
            continue
        if m == 0xD9:
            return 0, b""
        seg = (int(a[pos + 2]) << 8) | int(a[pos + 3])
        if m == 0xC4:
            i, end = pos + 4, min(pos + 2 + seg, n)
            while i + 17 <= end:
                have.add((int(a[i]) >> 4, int(a[i]) & 15))
                i += 17 + int(a[i + 1:i + 17].sum())
        elif m == 0xDA:
            ns = int(a[pos + 4]) if pos + 4 < n else 0
            sel = [int(a[pos + 6 + 2 * j]) for j in range(ns) if pos + 6 + 2 * j < n]
            need = {(0, t >> 4) for t in sel} | {(1, t & 15) for t in sel}
            miss = sorted((th, tc) for tc, th in need if th < 2 and (tc, th) not in have)
            out = b"".join(b"\xff\xc4" + (3 + len(_ANNEX_K[(tc, th)])).to_bytes(2, "big") + bytes([tc << 4 | th]) + _ANNEX_K[(tc, th)]
                           for th, tc in miss)
            return (pos, out) if out else (0, b"")
        pos += 2 + seg
    return 0, b""


def with_default_tables(data) -> bytes:
    """The JPEG file `data` with `default_tables` inserted (the same bytes when none is missing)."""
    at, seg = default_tables(data)
    b = bytes(data)
    return b[:at] + seg + b[at:] if seg else b


class MjpegSplitter:
    """Cuts a byte stream of concatenated JPEG files (`ffmpeg -c:v copy -f mjpeg -`, an MJPEG .avi or HTTP camera through
    ffmpeg) into whole files.  A file is found by its marker segments, walked by their lengths, so an APP1 Exif segment
    holding a thumbnail JPEG with its own SOI/EOI is skipped whole; after each SOS the entropy-coded data is scanned for
    the next marker that is not a stuffed FF 00, an RSTn or an FF fill byte, and segments are walked on from there until
    EOI (progressive and multi-scan files come out whole).  Bytes before an SOI are skipped; a new SOI before EOI
    abandons the file it interrupts.  The scans are vectorised (numpy) over the bytes read since the last call.

    `read(stream, dst)` reads the next file into the uint8 array `dst`; bytes read past its end are kept and start the
    next file.  A file longer than `dst` is skipped whole and counted in `dropped`."""

    SEEK, MARKERS, ENTROPY = 0, 1, 2
    WINDOW = 1 << 16                                               # bytes per vectorised scan

    def __init__(self):
        self.dropped = 0
        self.reset()

    def reset(self):
        """Forget any partial file and the bytes read past the last one (a reopened stream starts clean)."""
        self._carry = b""
        self._phase, self._pos = self.SEEK, 0

    def _scan(self, a, n) -> int:
        """Advance over a[:n] (a file starts at 0 once past SEEK) -> the file's end, or -1 when more bytes are needed.
        -2: an SOI is at _pos (after garbage, or interrupting the file in progress)."""
        while True:
            p = self._pos
            e = min(n - 1, p + self.WINDOW)                       # scan in windows: a marker is usually near
            if self._phase == self.SEEK:
                ff = np.flatnonzero(a[p:e] == 0xFF) + p
                hit = ff[a[ff + 1] == 0xD8]
                if len(hit) == 0:
                    self._pos = max(p, e)
                    if e < n - 1:
                        continue
                    return -1
                self._pos = int(hit[0])
                return -2
            if self._phase == self.ENTROPY:
                ff = np.flatnonzero(a[p:e] == 0xFF) + p
                nx = a[ff + 1]
                hit = ff[(nx != 0) & (nx != 0xFF) & ((nx < 0xD0) | (nx > 0xD7))]
                if len(hit) == 0:
                    self._pos = max(p, e)
                    if e < n - 1:
                        continue
                    return -1
                self._pos, self._phase = int(hit[0]), self.MARKERS
                continue
            if p + 2 > n:
                return -1
            if a[p] != 0xFF:                                       # not a marker where one must be: resynchronise
                self._phase = self.SEEK
                continue
            m = int(a[p + 1])
            if m == 0xFF:
                self._pos = p + 1
            elif m == 0xD9:
                return p + 2
            elif m == 0xD8:                                        # a new file interrupts this one
                return -2
            elif m == 0x01 or 0xD0 <= m <= 0xD7:
                self._pos = p + 2
            else:
                if p + 4 > n:
                    return -1
                self._pos = p + 2 + ((int(a[p + 2]) << 8) | int(a[p + 3]))
                if m == 0xDA:
                    self._phase = self.ENTROPY
                    if self._pos > n:
                        return -1
                elif self._pos > n:
                    return -1

    def read(self, stream, dst) -> int:
        """Read the next whole file of `stream` into dst[:n] and return n; 0 at the end of the stream (a partial file is
        then discarded).  Reads with readinto1 where the stream has it, so a live camera's frame is returned as soon as
        its last byte arrives."""
        rd = getattr(stream, "readinto1", None) or stream.readinto
        view, cap = memoryview(dst), len(dst)
        n = len(self._carry)
        dst[:n] = np.frombuffer(self._carry, np.uint8)
        self._carry = b""
        over = False                                               # the file in progress does not fit: drop it
        while True:
            e = self._scan(dst, n) if n else -1
            if e == -2:                                            # an SOI at _pos: move its file to the front
                d = self._pos
                dst[:n - d] = dst[d:n].copy()
                n -= d
                self._pos, self._phase, over = 2, self.MARKERS, False
                continue
            if e >= 0:
                if not over:
                    self._carry = dst[e:n].tobytes()
                    self._phase, self._pos = self.SEEK, 0
                    return e
                dst[:n - e] = dst[e:n].copy()                      # the dropped file ends here
                n -= e
                self._phase, self._pos, over = self.SEEK, 0, False
                continue
            if n == cap:                                           # full: keep only what the scan still needs
                if self._phase != self.SEEK and not over:
                    over = True
                    self.dropped += 1
                d = min(self._pos, n)
                dst[:n - d] = dst[d:n].copy()
                n -= d
                self._pos -= d
            got = rd(view[n:cap])
            if not got:
                self._phase, self._pos = self.SEEK, 0
                return 0
            n += got


class FrameMailbox:
    def __init__(self, height: int, width: int, pin: Optional[bool] = None, pix_fmt: str = BGR24):
        """height, width: the picture size in pixels; pix_fmt: "bgr24" (slots [H,W,3]) or "yuv420p" (slots [H*3/2,W],
        H and W even)."""
        self.height, self.width, self.pix_fmt = int(height), int(width), check_pix_fmt(pix_fmt)
        shape = (self.height, self.width, 3) if pix_fmt == BGR24 else (yuv420p_rows(self.height, self.width), self.width)
        self.frame_bytes = shape[0] * shape[1] * (shape[2] if len(shape) == 3 else 1)        # clearcam.py:403 for bgr24
        pin = torch.cuda.is_available() if pin is None else pin
        self._slots = torch.empty((3,) + shape, dtype=torch.uint8, pin_memory=pin)
        self._views = [memoryview(self._slots[i].numpy()).cast("B") for i in range(3)]
        self._lock = threading.Lock()
        self._latest = -1          # slot of the newest complete frame
        self._held = -1            # slot last handed to the consumer
        self.frame_num = -1        # clearcam.py:419

    def fill(self, stream) -> bool:
        """Read exactly one frame from `stream` into a free slot and publish it.  False on a short read / end of stream
        (nothing is published: the reference would raise on the reshape and retry, clearcam.py:418-421)."""
        with self._lock:
            slot = next(i for i in range(3) if i != self._latest and i != self._held)
        view, got = self._views[slot], 0
        while got < self.frame_bytes:
            n = stream.readinto(view[got:])
            if not n:
                return False
            got += n
        with self._lock:
            self._latest = slot
            self.frame_num += 1
        return True

    def latest(self, last_seen: int = -1) -> Optional[Tuple[int, torch.Tensor]]:
        """(frame_num, pinned uint8 view: [H,W,3] bgr24 or [H*3/2,W] yuv420p) of the newest frame, or None when there is none newer than `last_seen`
        (clearcam.py:446 `if frame_num == last_frame_num: return`).  The view stays intact until `latest` is called again."""
        with self._lock:
            if self._latest < 0 or self.frame_num == last_seen:
                return None
            self._held = self._latest
            return self.frame_num, self._slots[self._latest]


class JpegMailbox:
    """The FrameMailbox of a Motion-JPEG camera (`-c:v copy -f mjpeg`): three pinned slots, each holding one whole JPEG
    file, with FrameMailbox's rules (one being written, one published, one possibly still held by the consumer).  A slot
    holds height*width*3 bytes (a bgr24 frame, so an MJPEG camera pins no more than a bgr24 one) plus room for the DHT
    segments `default_tables` inserts; a file that does not fit is dropped and counted in `dropped`."""

    pix_fmt = MJPEG

    def __init__(self, height: int, width: int, pin: Optional[bool] = None):
        self.height, self.width = int(height), int(width)
        if self.height <= 0 or self.width <= 0:
            raise ValueError(f"bad picture size {width}x{height}")
        self.capacity = self.height * self.width * 3 + TABLE_ROOM
        pin = torch.cuda.is_available() if pin is None else pin
        self._slots = torch.empty((3, self.capacity), dtype=torch.uint8, pin_memory=pin)
        self._arrays = [self._slots[i].numpy() for i in range(3)]
        self._len = [0, 0, 0]
        self._splitter = MjpegSplitter()
        self._stream = None
        self._lock = threading.Lock()
        self._latest = -1
        self._held = -1
        self.frame_num = -1

    @property
    def dropped(self) -> int:
        """Files skipped because they were larger than a slot."""
        return self._splitter.dropped

    def fill(self, stream) -> bool:
        """Read one whole JPEG file from `stream` into a free slot, insert the Huffman tables its scan lacks
        (`default_tables`) and publish it.  False at the end of the stream (nothing is published).  A stream other than
        the last one starts clean: bytes kept from the old stream are dropped."""
        if stream is not self._stream:
            self._splitter.reset()
            self._stream = stream
        with self._lock:
            slot = next(i for i in range(3) if i != self._latest and i != self._held)
        a = self._arrays[slot]
        n = self._splitter.read(stream, a[:self.capacity - TABLE_ROOM])
        if not n:
            return False
        at, seg = default_tables(a[:n])
        if seg:
            a[at + len(seg):n + len(seg)] = a[at:n].copy()
            a[at:at + len(seg)] = np.frombuffer(seg, np.uint8)
            n += len(seg)
        with self._lock:
            self._len[slot] = n
            self._latest = slot
            self.frame_num += 1
        return True

    def latest(self, last_seen: int = -1) -> Optional[Tuple[int, torch.Tensor]]:
        """(frame_num, pinned uint8 [n] view of the newest file's bytes), or None when there is none newer than
        `last_seen`.  The view stays intact until `latest` is called again."""
        with self._lock:
            if self._latest < 0 or self.frame_num == last_seen:
                return None
            self._held = self._latest
            return self.frame_num, self._slots[self._latest][:self._len[self._latest]]


class PipeReader(threading.Thread):
    def __init__(self, mailbox: FrameMailbox, open_stream: Callable[[], object], max_fail: int = 5, retry_sleep: float = 0.5,
                 name: str = "camera"):
        super().__init__(daemon=True, name=f"ingest-{name}")
        self.mailbox, self.open_stream, self.max_fail, self.retry_sleep = mailbox, open_stream, max_fail, retry_sleep
        self.restarts = 0
        self.open_errors = 0                   # failed open_stream() calls (camera / ffmpeg down): retried with back-off
        self.last_error: Optional[BaseException] = None
        self._stream = None
        self._stop_evt = threading.Event()

    def stop(self):
        """Ask the thread to end and close the stream so a read blocked on a silent camera returns."""
        self._stop_evt.set()
        self._close()

    def _close(self):
        s, self._stream = self._stream, None
        if s is not None:
            try:
                s.close()
            except Exception:
                pass

    def _open(self) -> bool:
        """open_stream() under supervision: a camera or ffmpeg that is down must not kill the reader thread (the reference's
        frame_loop keeps logging and retrying, clearcam.py:401-421).  Back-off doubles up to 8x retry_sleep."""
        delay = self.retry_sleep
        while not self._stop_evt.is_set():
            try:
                self._stream = self.open_stream()
                return True
            except Exception as ex:
                self.open_errors += 1
                self.last_error = ex
                self._stop_evt.wait(delay)
                delay = min(delay * 2, self.retry_sleep * 8)
        return False

    def run(self):
        fails = 0
        try:
            if not self._open():
                return
            while not self._stop_evt.is_set():
                try:
                    ok = self.mailbox.fill(self._stream)
                except Exception as ex:                             # clearcam.py:420-421: log-and-retry supervision
                    self.last_error = ex
                    ok = False
                if ok:
                    fails = 0
                    continue
                if self._stop_evt.is_set():
                    break
                fails += 1
                if fails > self.max_fail:                           # clearcam.py:408-411: restart the stream
                    self._close()
                    if not self._open():
                        break
                    fails = 0
                    self.restarts += 1
                self._stop_evt.wait(self.retry_sleep)
        finally:
            self._close()


class VideoReader:
    """A recorded video read from a rawvideo byte stream (e.g. `ffmpeg -i video.mp4 -f rawvideo -pix_fmt bgr24 -`) in runs of
    up to `run` frames.  Unlike FrameMailbox nothing is dropped: frames come in order.  With every=2 the first frame of each
    pair is skipped and the second kept (0-based frames 1, 3, 5, ...), as the reference's `grab()` + `read()` per step
    does (clearcam.py:431-432).  A thread fills two alternating pinned run buffers; iterating yields (frames, positions):
    frames a pinned uint8 view [n,H,W,3] (bgr24) or [n,H*3/2,W] (yuv420p), or with pix_fmt="mjpeg" (a stream of JPEG
    files, `ffmpeg -i video.avi -c:v copy -f mjpeg -`) a list of n pinned uint8 views, one JPEG file each with its
    default Huffman tables inserted (files larger than height*width*3 bytes are skipped and not counted as frames), all
    valid until the next run is asked for, and
    positions the (n,) int64 CAP_PROP_POS_FRAMES of each frame (its 0-based index + 1), from which the caller computes
    video time (pos / fps) and progress (pos / frame count).  The last run may be short; reading ends at the end of the
    stream or at a short read (a partial last frame is dropped).  An exception raised while reading is raised by the
    iteration, after the runs read before it.  `close()` (or leaving a `with` block) ends the thread of a reader the caller
    stops using early."""

    def __init__(self, stream, height: int, width: int, pix_fmt: str = BGR24, run: int = 32, every: int = 2, pin: Optional[bool] = None):
        if run < 1 or every < 1:
            raise ValueError("run and every must be >= 1")
        self.mjpeg = pix_fmt == MJPEG
        self.height, self.width, self.pix_fmt = int(height), int(width), pix_fmt if self.mjpeg else check_pix_fmt(pix_fmt)
        shape = (self.height, self.width, 3) if self.pix_fmt in (BGR24, MJPEG) else \
            (yuv420p_rows(self.height, self.width), self.width)
        self.frame_bytes = int(np.prod(shape))
        pin = torch.cuda.is_available() if pin is None else pin
        if self.mjpeg:                               # one JPEG file per bgr24 frame's bytes, plus room for its tables
            self.capacity = self.frame_bytes + TABLE_ROOM
            self._splitter = MjpegSplitter()
            self._bufs = [torch.empty(run * self.capacity, dtype=torch.uint8, pin_memory=pin) for _ in range(2)]
            self._skip = np.empty(self.capacity - TABLE_ROOM, np.uint8)
        else:
            self._bufs = [torch.empty((run,) + shape, dtype=torch.uint8, pin_memory=pin) for _ in range(2)]
            self._skip = bytearray(self.frame_bytes)
        self.stream, self.run, self.every = stream, int(run), int(every)
        self._free = queue.Queue()                    # buffer indices the reader may fill
        self._full = queue.Queue()                    # (buffer, n, positions) runs, None at the end
        self._free.put(0)
        self._free.put(1)
        self._held = None                             # buffer last handed to the consumer
        self._stop = threading.Event()
        self.error: Optional[BaseException] = None
        self._thread = threading.Thread(target=self._read, daemon=True, name="video-reader")
        self._thread.start()

    def _fill(self, view) -> bool:
        got = 0
        while got < self.frame_bytes:
            n = self.stream.readinto(view[got:])
            if not n:
                return False
            got += n
        return True

    def _fill_jpeg(self, a) -> int:
        """The next JPEG file into a[:n] with its default tables (n returned), 0 at the end of the stream."""
        n = self._splitter.read(self.stream, a[:len(a) - TABLE_ROOM])
        if n:
            at, seg = default_tables(a[:n])
            if seg:
                a[at + len(seg):n + len(seg)] = a[at:n].copy()
                a[at:at + len(seg)] = np.frombuffer(seg, np.uint8)
                n += len(seg)
        return n

    def _read_jpeg(self):
        index = 0
        try:
            while True:
                b = self._free.get()
                if self._stop.is_set():
                    break
                a = self._bufs[b].numpy()
                pos, spans, end = [], [], False
                while len(pos) < self.run and not self._stop.is_set():
                    for _ in range(self.every - 1):
                        if not self._splitter.read(self.stream, self._skip):
                            end = True
                            break
                        index += 1
                    o = len(pos) * self.capacity
                    n = 0 if end else self._fill_jpeg(a[o:o + self.capacity])
                    if not n:
                        end = True
                        break
                    index += 1
                    pos.append(index)
                    spans.append((o, n))
                if pos:
                    self._full.put((b, np.array(pos, np.int64), spans))
                if end:
                    break
        except BaseException as ex:
            self.error = ex
        finally:
            self._full.put(None)

    def _read(self):
        if self.mjpeg:
            return self._read_jpeg()
        index = 0                                     # frames read from the stream so far
        try:
            while True:
                b = self._free.get()
                if self._stop.is_set():
                    break
                views = memoryview(self._bufs[b].numpy()).cast("B")
                pos, end = [], False
                while len(pos) < self.run and not self._stop.is_set():
                    for _ in range(self.every - 1):   # grab(): skipped
                        if not self._fill(memoryview(self._skip)):
                            end = True
                            break
                        index += 1
                    if end or not self._fill(views[len(pos) * self.frame_bytes:(len(pos) + 1) * self.frame_bytes]):
                        end = True
                        break
                    index += 1
                    pos.append(index)
                if pos:
                    self._full.put((b, np.array(pos, np.int64)))
                if end:
                    break
        except BaseException as ex:                   # reported to the consumer, which then ends
            self.error = ex
        finally:
            self._full.put(None)

    def __iter__(self):
        return self

    def __next__(self) -> Tuple[torch.Tensor, np.ndarray]:
        if self._held is not None:                    # the previous run's buffer may be refilled now
            self._free.put(self._held)
            self._held = None
        got = self._full.get()
        if got is None:
            self._full.put(None)
            if self.error is not None:
                raise self.error
            raise StopIteration
        b, pos = got[:2]
        self._held = b
        if self.mjpeg:
            return [self._bufs[b][o:o + n] for o, n in got[2]], pos
        return self._bufs[b][:len(pos)], pos

    def close(self):
        """End the reader thread (a run in progress is dropped) and wait for it."""
        self._stop.set()
        self._free.put(-1)                            # wakes a thread waiting for a buffer
        self._thread.join()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
