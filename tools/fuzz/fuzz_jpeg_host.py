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
# PNG streams (every colour type, Adam7, split IDAT runs, eXIf): the chunk walk of the planner
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "tests"))
import png_streams
seeds += [bytearray(s) for _, s in png_streams.corpus()[::6]]
# TIFF streams (strips, tiles, planes, both byte orders, every codec): the IFD walk and the segment table of the planner
import tiff_streams
seeds += [bytearray(s) for _, s in tiff_streams.corpus()[::8]]
# WebP streams (simple and VP8X, alpha, EXIF, every partition count, simple and normal filter): the RIFF walk and the VP8 header parse.
# Written by Pillow and libwebp's encoder only: cv2's WebP encoder throws (and catches) C++ exceptions, which the preloaded ASAN
# runtime cannot intercept in cv2's module
import webp_streams
wimg = [np.random.default_rng(k).integers(0, 256, (h, w, 3), dtype=np.uint8) for k, (h, w) in enumerate([(1, 1), (17, 33), (40, 56)])]
seeds += [bytearray(webp_streams.pil_webp(a, quality=q, method=m)) for a in wimg for q, m in ((20, 0), (90, 4))]
seeds += [bytearray(webp_streams.pil_webp(np.dstack([wimg[1], wimg[1][..., 0]]), quality=60)),
          bytearray(webp_streams.pil_webp(wimg[2], quality=60, exif=webp_streams.exif_orientation(6)))]
if webp_streams.libwebp():
    seeds += [bytearray(webp_streams.libwebp_encode(wimg[2], 60.0, partitions=3, method=2, filter_type=t)) for t in (0, 1)]
# BMP and PNM streams (every header size, palettes, bitfields, RLE4 / RLE8, P1 - P6, comments): the header parse of the planner
import bitmap_streams
seeds += [bytearray(s) for n, s in bitmap_streams.corpus() if len(s) < 100000][::7]
# lossless JPEG streams (SOF3: predictors, point transforms, restart intervals, tables with codes up to 16 bits): the frame checks, the
# table build and the split at the restart markers of ljpeg_plan.h
import ljpeg_streams
seeds += [bytearray(s) for n, s, _, _ in ljpeg_streams.corpus() if len(s) < 100000][::5]
# WAV and FLAC streams (every format the corpus holds, the refused and the corrupt ones): the container parse, plan set-up and the
# launch-side staging and descriptor build of decoders.audio (audio_decode_plan.h, dalib200AudioPlanSetup / dalib200AudioLaunch)
import audio_streams
audio_seeds = [bytearray(s) for _, s, _, _ in audio_streams.corpus() if len(s) < 60000] + \
    [bytearray(s) for _, s, _, _ in audio_streams.refused()] + [bytearray(s) for _, s in audio_streams.corrupt()]
audio_plan = C.c_void_p()
assert L.dalib200AudioPlanCreate(C.byref(audio_plan), 4) == 0, L.dalib200GetLastError()
ainfo = (C.c_int32 * 8)()
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
    # an audio batch: RIFF chunk sizes, fmt fields, ID3 sizes, metadata block headers and STREAMINFO fields mutated like the above
    abatch = []
    for b in range(int(rng.integers(1, 4))):
        s = bytearray(audio_seeds[int(rng.integers(0, len(audio_seeds)))])
        k = int(rng.integers(0, 4))
        if k == 0:
            for _ in range(rng.integers(1, 6)): s[rng.integers(0, min(len(s), 120))] = rng.integers(0, 256)
        elif k == 1:
            s = s[:rng.integers(0, len(s))]
        elif k == 2:
            p = rng.integers(0, len(s)); s[p:p] = bytes(rng.integers(0, 256, rng.integers(1, 9)).astype(np.uint8))
        abatch.append(bytes(s) if len(s) else b"\0")
    abufs = [(C.c_uint8 * len(s)).from_buffer_copy(s) for s in abatch]
    aptrs = (C.c_void_p * len(abufs))(*[C.addressof(b) for b in abufs])
    alens = (C.c_size_t * len(abufs))(*[len(s) for s in abatch])
    aprm = (C.c_int32 * (4 * len(abufs)))()
    for b in range(len(abufs)):
        L.dalib200AudioGetInfo(abufs[b], C.c_size_t(len(abatch[b])), ainfo)
        rate = float(rng.choice([0.0, 16000.0, 8000.5, -1.0]))
        aprm[4 * b:4 * b + 4] = [int(rng.integers(0, 2)), C.c_int32.from_buffer(C.c_float(rate)).value, C.c_int32.from_buffer(C.c_float(50.0)).value,
                                 int(rng.choice([9, 5, 6, 1]))]
    rc = L.dalib200AudioPlanSetup(audio_plan, len(abufs), aptrs, alens, aprm)
    if rc == 0:
        shape, nd, r = (C.c_int64 * 2)(), C.c_int32(), C.c_float()
        for b in range(len(abufs)):
            L.dalib200AudioPlanGetOutputShape(audio_plan, b, shape, C.byref(nd), C.byref(r))
        outs = (C.c_void_p * len(abufs))(*[0x10000 * (b + 1) for b in range(len(abufs))])       # never dereferenced on the host
        rc2 = L.dalib200AudioLaunch(audio_plan, outs, outs, None)
        rcs["audio launch", rc2] = rcs.get(("audio launch", rc2), 0) + 1
    rcs["audio", rc] = rcs.get(("audio", rc), 0) + 1
print("seed", sys.argv[2] if len(sys.argv) > 2 else 0, "iterations", n, "status histogram", rcs, "- no sanitizer report")
