#!/bin/bash
# tools/fuzz/run.sh [iterations] [seeds...] -- fuzzes the HOST side of the JPEG decoder (marker / EXIF / table parsing, restart-marker scan,
# ROI and descriptor build of dalib200JpegGetInfo / dalib200JpegPlanSetupEx) under AddressSanitizer, without a GPU: jpeg.cu + common.cu
# are built with -fsanitize=address and the handful of CUDA runtime calls the host side makes are replaced by a preloaded stub
# (cuda_stub.c: events = no-ops, pinned / device allocations = malloc, so that ASAN's red zones surround them).
# Inputs: valid baseline and progressive streams (4:2:0 / 4:4:4 / 4:2:2 / gray / CMYK / YCCK, restart intervals, EXIF orientations), PNG, TIFF, WebP, BMP and PNM streams with byte flips, truncation,
# and WAV / FLAC streams through the audio decoder's container parse, plan set-up and launch-side staging (dalib200Audio*),
# corrupted segment lengths, wrapping EXIF offsets, inserted / deleted bytes, markers sprinkled into the entropy data.
# A finding is an ASAN report on stderr (non-zero exit).
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"; ROOT="$(cd "$HERE/../.." && pwd)"
OUT="${FUZZ_DIR:-/tmp/dali_b200_fuzz}"; mkdir -p "$OUT"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
F="-gencode arch=compute_90a,code=sm_90a -O1 -g -std=c++17 -Xcompiler -fPIC,-fsanitize=address,-fno-omit-frame-pointer --expt-relaxed-constexpr -fmad=false -I$ROOT/include"
$NVCC $F -c "$ROOT/dali_b200/csrc/jpeg.cu" -o "$OUT/jpeg.o"
$NVCC $F -c "$ROOT/dali_b200/csrc/common.cu" -o "$OUT/common.o"
$NVCC $F -c "$ROOT/dali_b200/csrc/jpeg_prog.cu" -o "$OUT/jpeg_prog.o"
$NVCC $F -c "$ROOT/dali_b200/csrc/png.cu" -o "$OUT/png.o"
$NVCC $F -c "$ROOT/dali_b200/csrc/tiff.cu" -o "$OUT/tiff.o"
$NVCC $F -c "$ROOT/dali_b200/csrc/webp.cu" -o "$OUT/webp.o"
$NVCC $F -c "$ROOT/dali_b200/csrc/bitmap.cu" -o "$OUT/bitmap.o"
$NVCC $F -c "$ROOT/dali_b200/csrc/ljpeg.cu" -o "$OUT/ljpeg.o"
$NVCC $F -c "$ROOT/dali_b200/csrc/audio_decode.cu" -o "$OUT/audio_decode.o"
$NVCC $F -c "$ROOT/dali_b200/csrc/audio_tail.cu" -o "$OUT/audio_tail.o"
$NVCC -shared -o "$OUT/libfuzz.so" "$OUT/jpeg.o" "$OUT/common.o" "$OUT/jpeg_prog.o" "$OUT/png.o" "$OUT/tiff.o" "$OUT/webp.o" "$OUT/bitmap.o" "$OUT/ljpeg.o" "$OUT/audio_decode.o" "$OUT/audio_tail.o" -gencode arch=compute_90a,code=sm_90a -lcudart -Xcompiler -fsanitize=address
gcc -shared -fPIC -O1 -o "$OUT/cuda_stub.so" "$HERE/cuda_stub.c"
# the progressive scan decoder itself (the body of prog_scan_kernel, compiled for the host by tools/emul) under ASAN + UBSAN on mutated
# progressive streams: garbage Huffman codes, runs past the band, truncated scans, markers inside the data must stay inside the arena
g++ -std=c++17 -O1 -g -fsanitize=address,undefined -fno-omit-frame-pointer -shared -fPIC -I/usr/local/cuda/include \
    "$ROOT/tools/emul/jpeg_prog_emul.cc" -o "$OUT/libjpegprog_asan.so"
N="${1:-15000}"; shift || true
SEEDS="${*:-1 2 3}"
for s in $SEEDS; do
  LD_PRELOAD="$(gcc -print-file-name=libasan.so) $OUT/cuda_stub.so" ASAN_OPTIONS=detect_leaks=0 python "$HERE/fuzz_jpeg_host.py" "$OUT/libfuzz.so" "$s" "$N"
  LD_PRELOAD="$(gcc -print-file-name=libasan.so)" ASAN_OPTIONS=detect_leaks=0 UBSAN_OPTIONS=halt_on_error=1:print_stacktrace=1 \
    python "$HERE/fuzz_jpeg_prog_emul.py" "$OUT/libjpegprog_asan.so" "$s" "$((N / 4))"
done
