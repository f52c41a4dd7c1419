"""Image decode process of the sharded loader (`make_dataset(decode_processes=N)`): run BY PATH (`python _decode_worker.py
<address> <slot>`), imports only numpy + PIL - never the framework / torch - so a hundred of them start in about a second.

Why processes: PIL releases the GIL inside the JPEG decoder and the resampler, but the Python part of opening an image
(marker parsing in JpegImagePlugin, BytesIO, the final array copy) holds it for ~0.2 ms per image - decode THREADS of one
process top out at a few thousand images/s no matter how many cores there are - below what one GPU trains on.

Protocol (binary frames over the authenticated unix socket, no pickling):
    request : int32[3 + n] = (H, W, n, len_0 .. len_{n-1})  followed by the n payloads back to back;  an EMPTY frame = exit
    reply   : uint8[n, H, W, 3] (decoded, RGB, bilinear resize to HxW - the same operations as models.preprocess.decode_image)
"""
import io
import os
import sys
from multiprocessing.connection import Client

import numpy as np


def decode_into(out: np.ndarray, payload, h: int, w: int) -> None:
    if len(payload) == h * w * 3:   # raw uint8 image of exactly the target size (synthetic tables): no decoder
        out[...] = np.frombuffer(payload, dtype=np.uint8).reshape(h, w, 3)
        return
    from PIL import Image

    img = Image.open(io.BytesIO(payload)).convert("RGB")
    if img.size != (w, h):
        img = img.resize((w, h), Image.BILINEAR)
    out[...] = np.asarray(img, dtype=np.uint8)


def serve(conn) -> None:
    while True:
        try:
            frame = conn.recv_bytes()
        except EOFError:
            return
        if not frame:
            return
        head = np.frombuffer(frame, dtype=np.int32, count=3)
        h, w, n = int(head[0]), int(head[1]), int(head[2])
        lens = np.frombuffer(frame, dtype=np.int32, count=n, offset=12)
        out = np.empty((n, h, w, 3), dtype=np.uint8)
        view = memoryview(frame)
        off = 12 + 4 * n
        for i in range(n):
            decode_into(out[i], view[off:off + int(lens[i])], h, w)
            off += int(lens[i])
        conn.send_bytes(memoryview(out).cast("B"))


if __name__ == "__main__":
    os.environ.setdefault("OMP_NUM_THREADS", "1")
    conn = Client(sys.argv[1], family="AF_UNIX", authkey=bytes.fromhex(os.environ["B200DDL_PP_KEY"]))
    try:
        serve(conn)
    except (BrokenPipeError, ConnectionResetError, KeyboardInterrupt):
        pass
