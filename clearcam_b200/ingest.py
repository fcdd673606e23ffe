"""Frame ingest for the batched detector (SURVEY.md §8f N4): raw frames from a pipe into pinned host memory.

The reference reads `width*height*3` bytes per frame from an ffmpeg `-f rawvideo -pix_fmt bgr24` pipe into a fresh
bytes object, wraps it in numpy, and the consumer copies it again before use (`frame_loop`, clearcam.py:401-421;
`process_frame` :446-447).  Here the bytes land once, in a page-locked slot the GPU can DMA from:

  * `FrameMailbox`   one camera's latest frame (the reference's `raw_frame[cam]` / `frame_num[cam]`), three pinned slots:
                     one being written, one published, one possibly still held by the consumer — no copy, no tearing
  * `PipeReader`     the `frame_loop` thread: fill the mailbox from a byte stream, count short reads and reopen the stream
                     after more than five in a row (clearcam.py:407-412)
  * `CameraBatch.step_mailboxes` (cameras.py) takes every camera's unseen frame straight from its mailbox

Frames are bgr24 (`-pix_fmt bgr24`, H*W*3 bytes) or, with `FrameMailbox(h, w, pix_fmt="yuv420p")`, yuv420p
(`-pix_fmt yuv420p`, H*W*3/2 bytes: half the pipe, pinned-memory and PCIe bytes, and no swscale conversion on the host;
the GPU converts them, see clearcam_b200/pixfmt.py).

Spawning ffmpeg (and HLS recording, clearcam.py:310-371) stays with the caller: `PipeReader` takes any callable that
returns a readable binary stream, e.g. `lambda: subprocess.Popen(cmd, stdout=subprocess.PIPE).stdout`."""
import threading
import time
from typing import Callable, Optional, Tuple

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
