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

Spawning ffmpeg (and HLS recording, clearcam.py:310-371) stays with the caller: `PipeReader` takes any callable that
returns a readable binary stream, e.g. `lambda: subprocess.Popen(cmd, stdout=subprocess.PIPE).stdout`."""
import queue
import threading
import time
from typing import Callable, Optional, Tuple

import numpy as np

import torch

from .pixfmt import BGR24, check_pix_fmt, yuv420p_rows


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
    frames a pinned uint8 view [n,H,W,3] (bgr24) or [n,H*3/2,W] (yuv420p), valid until the next run is asked for, and
    positions the (n,) int64 CAP_PROP_POS_FRAMES of each frame (its 0-based index + 1), from which the caller computes
    video time (pos / fps) and progress (pos / frame count).  The last run may be short; reading ends at the end of the
    stream or at a short read (a partial last frame is dropped).  An exception raised while reading is raised by the
    iteration, after the runs read before it.  `close()` (or leaving a `with` block) ends the thread of a reader the caller
    stops using early."""

    def __init__(self, stream, height: int, width: int, pix_fmt: str = BGR24, run: int = 32, every: int = 2, pin: Optional[bool] = None):
        if run < 1 or every < 1:
            raise ValueError("run and every must be >= 1")
        self.height, self.width, self.pix_fmt = int(height), int(width), check_pix_fmt(pix_fmt)
        shape = (self.height, self.width, 3) if self.pix_fmt == BGR24 else (yuv420p_rows(self.height, self.width), self.width)
        self.frame_bytes = int(np.prod(shape))
        pin = torch.cuda.is_available() if pin is None else pin
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

    def _read(self):
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
        b, pos = got
        self._held = b
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
