"""Host-side fuzzer of the JPEG decoder plan (see run.sh): python fuzz_jpeg_host.py <libfuzz.so> <seed> <iterations>."""
import ctypes as C, numpy as np, sys, cv2, os
L = C.CDLL(sys.argv[1])
L.dalib200GetLastError.restype = C.c_char_p
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
from oracle import pyoracle as po
rng = np.random.default_rng(int(sys.argv[2]) if len(sys.argv) > 2 else 0)
def synth(h, w, q=90, sub=None, rst=0, gray=False, prog=False):
    img = rng.integers(0, 255, (h, w) if gray else (h, w, 3)).astype(np.uint8)
    p = [cv2.IMWRITE_JPEG_QUALITY, q] + ([cv2.IMWRITE_JPEG_PROGRESSIVE, 1] if prog else [])
    if sub is not None: p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sub]
    if rst: p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    ok, e = cv2.imencode(".jpg", img, p)
    return bytearray(e.tobytes())
seeds = [synth(33, 47), synth(64, 64, sub=cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444), synth(40, 24, rst=2), synth(17, 19, gray=True), synth(48, 80, rst=1, sub=cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422)]
seeds += [bytearray(po.with_exif_orientation(bytes(seeds[0]), o)) for o in (3, 6, 8)]
seeds += [synth(33, 47, prog=True), synth(40, 24, rst=2, prog=True), synth(17, 19, gray=True, prog=True),
          synth(48, 40, sub=cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, prog=True)]
# 4-component streams (CMYK, YCCK, no Adobe marker; baseline and progressive; 4:4:4 and subsampled), written by Pillow
cmyk = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "tests", "golden", "jpeg_cmyk.npz"))
seeds += [bytearray(cmyk[f"enc_{k}"].tobytes()) for k in range(len(cmyk.files) // 4) if str(cmyk[f"name_{k}"]).endswith("61x77")]
info = (C.c_int32 * 32)()
plan = C.c_void_p()
assert L.dalib200JpegPlanCreate(C.byref(plan), 4) == 0, L.dalib200GetLastError()
n = int(sys.argv[3]) if len(sys.argv) > 3 else 5000
rcs = {}
for it in range(n):
    batch = []
    for b in range(int(rng.integers(1, 4))):
        s = bytearray(seeds[int(rng.integers(0, len(seeds)))])
        k = int(rng.integers(0, 7))
        if k == 0:
            for _ in range(rng.integers(1, 6)): s[rng.integers(0, len(s))] = rng.integers(0, 256)
        elif k == 1:
            s = s[:rng.integers(0, len(s))]
        elif k == 2:
            pos = [i for i in range(2, len(s) - 3) if s[i] == 0xFF and s[i + 1] not in (0, 0xFF) and not 0xD0 <= s[i + 1] <= 0xD9]
            if pos:
                p = pos[rng.integers(0, len(pos))]; v = int(rng.choice([0, 1, 2, 3, 0xFFFF, 0xFFFE, 0x7FFF, rng.integers(0, 65536)]))
                s[p + 2] = v >> 8; s[p + 3] = v & 255
        elif k == 3:   # sprinkle markers into the entropy data (restart / EOI / garbage markers)
            for _ in range(rng.integers(1, 5)):
                p = rng.integers(len(s) // 2, len(s) - 1); s[p] = 0xFF; s[p + 1] = int(rng.choice([0xD0, 0xD3, 0xD7, 0xD9, 0x00, 0xFF, 0xC4, 0xDA]))
        elif k == 4:
            p = rng.integers(0, len(s)); s[p:p] = bytes(rng.integers(0, 256, rng.integers(1, 9)).astype(np.uint8))
        elif k == 5:
            p = rng.integers(0, len(s)); del s[p:p + rng.integers(1, 9)]
        batch.append(bytes(s) if len(s) else b"\0")
    bufs = [(C.c_uint8 * len(s)).from_buffer_copy(s) for s in batch]
    ptrs = (C.c_void_p * len(bufs))(*[C.addressof(b) for b in bufs])
    lens = (C.c_size_t * len(bufs))(*[len(s) for s in batch])
    prm = (C.c_int32 * 4)(int(rng.integers(0, 4)), int(rng.integers(0, 2)), int(rng.choice([0, 9])), int(rng.integers(0, 2)))
    rois = None
    if rng.integers(0, 2):
        rois = (C.c_int32 * (6 * len(bufs)))()
        for b in range(len(bufs)):
            x0, y0 = int(rng.integers(-2, 40)), int(rng.integers(-2, 40))
            rois[6 * b:6 * b + 6] = [int(rng.integers(0, 2)), x0, y0, x0 + int(rng.integers(-1, 50)), y0 + int(rng.integers(-1, 50)), int(rng.integers(0, 2))]
    for b in range(len(bufs)):
        L.dalib200JpegGetInfo(bufs[b], C.c_size_t(len(batch[b])), info)
    rc = L.dalib200JpegPlanSetupEx(plan, len(bufs), ptrs, lens, prm, rois)
    if rc == 0:
        hwc = (C.c_int32 * 3)()
        outs = (C.c_void_p * len(bufs))(*[0x10000 * (b + 1) for b in range(len(bufs))])       # never dereferenced on the host
        for b in range(len(bufs)):
            L.dalib200JpegPlanGetOutputShape(plan, b, hwc)
        # the staging copy of the streams and the launch-side descriptor build (kernels are stubbed out)
        L.dalib200JpegPlanSetSourceStable(plan, int(rng.integers(0, 2)))
        rc2 = L.dalib200JpegUpload(plan, None)
        if rc2 == 0:
            rc2 = L.dalib200JpegLaunch(plan, outs, None)
        rcs["launch", rc2] = rcs.get(("launch", rc2), 0) + 1
    rcs[rc] = rcs.get(rc, 0) + 1
print("seed", sys.argv[2] if len(sys.argv) > 2 else 0, "iterations", n, "status histogram", rcs, "- no sanitizer report")
