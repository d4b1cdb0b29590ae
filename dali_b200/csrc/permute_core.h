// dali_b200/csrc/permute_core.h -- the per-thread bodies of the batched N-D strided copy behind fn.transpose, fn.cat and fn.stack
// (csrc/permute.cu), written as host/device functions so that tools/emul/permute_emul.cc runs the very code the device runs.
//
// One descriptor (PermDesc, built by csrc/permute_plan.h) copies one dense input sample into its place in an output sample.  Its
// dimensions are already collapsed; two paths read them:
//   ROW    the contiguous run shared by both sides is at least kPermRowBytes: rows of `r` bytes are copied as they are, a work item
//          being up to kPermTileBytes of whole rows or one segment of a longer row.  Words of `w` bytes (16 when both sides are
//          16-byte aligned) with a byte-wise head and tail.
//   TILE   units of `r` bytes are exchanged between the input's fastest dimension X and the output's fastest dimension Y through a
//          shared-memory tile of tx x ty units: pieces of `ps` bytes (a power of two dividing r) are read in input order and written
//          in output order, so both sides move whole sectors.  The tile is held in input order ("in-major", rows of tx units) or,
//          when Y is the small dimension, in output order ("out-major", rows of ty units); a side whose tile rows are contiguous in
//          memory and in shared memory is moved as one span with 16-byte words where the addresses allow.  A padded row pitch (an
//          odd number of words) keeps the column-wise side free of bank conflicts.
// Every offset is 64-bit, so one sample may exceed 2^31 bytes; indices inside a work item are 32-bit.
#ifndef DALI_B200_CSRC_PERMUTE_CORE_H_
#define DALI_B200_CSRC_PERMUTE_CORE_H_

#include <stdint.h>
#include "host_device.h"

namespace dalib200 {

constexpr int kPermMaxDim = 6;
constexpr int kPermThreads = 256;
constexpr int kPermTileBytes = 16384;       // bytes of a TILE work item's shared-memory tile, and of a ROW work item
constexpr int kPermSmemBytes = kPermTileBytes;
enum : int32_t { kPermPathRow = 0, kPermPathTile = 1 };

#ifdef __CUDACC__
using PermV8 = uint2;
using PermV16 = uint4;
#else
struct PermV8 { uint32_t x, y; };
struct alignas(16) PermV16 { uint32_t x, y, z, w; };
#endif

struct PermDesc {
  const uint8_t *in; uint8_t *out;
  int64_t first_item, items;
  int64_t out_off;                                                  // byte offset of this input inside the output sample
  int64_t ext[kPermMaxDim], istr[kPermMaxDim], ostr[kPermMaxDim];   // outer dimensions in output order, byte strides
  int64_t nx, ny, istr_x, istr_y, ostr_x, ostr_y;                   // TILE: the exchanged dimensions
  int64_t r;                                                        // TILE: unit bytes; ROW: row bytes
  int64_t rows, rows_per_item, segs;                                // ROW
  int32_t path, nouter, tx, ty, ntx, nty;
  int32_t out_major, padded, align;                                 // align: power of two dividing every stride and r
  int32_t ps, pitch, w;                                             // set at launch from the pointers: piece, pitch, ROW word
};

// the byte offsets of outer index `o` on both sides
DB_HD void perm_outer(const PermDesc &d, int64_t o, int64_t *io, int64_t *oo) {
  int64_t a = 0, b = 0;
  for (int k = d.nouter - 1; k >= 0; k--) {
    const int64_t q = o / d.ext[k], idx = o - q * d.ext[k];
    a += idx * d.istr[k]; b += idx * d.ostr[k]; o = q;
  }
  *io = a; *oo = b;
}

// ---------------------------------------------------------------------------------------------------------------- spans
template <typename W>
DB_HD void perm_words(uint8_t *dst, const uint8_t *src, int64_t nwords, int tid, int nt) {
  for (int64_t i = tid; i < nwords; i += nt) reinterpret_cast<W *>(dst)[i] = reinterpret_cast<const W *>(src)[i];
}

// a contiguous span, in the widest words that both addresses and the length allow
DB_HD void perm_span(uint8_t *dst, const uint8_t *src, int64_t bytes, int tid, int nt) {
  const uint64_t a = (uint64_t)(uintptr_t)dst | (uint64_t)(uintptr_t)src | (uint64_t)bytes;
  if ((a & 15) == 0) perm_words<PermV16>(dst, src, bytes >> 4, tid, nt);
  else if ((a & 7) == 0) perm_words<PermV8>(dst, src, bytes >> 3, tid, nt);
  else if ((a & 3) == 0) perm_words<uint32_t>(dst, src, bytes >> 2, tid, nt);
  else if ((a & 1) == 0) perm_words<uint16_t>(dst, src, bytes >> 1, tid, nt);
  else perm_words<uint8_t>(dst, src, bytes, tid, nt);
}

// ---------------------------------------------------------------------------------------------------------------- TILE
struct PermTile {
  const uint8_t *in; uint8_t *out;
  int32_t cx, cy;                       // units of this tile along X and Y (edge tiles are partial)
};

DB_HD PermTile perm_tile_at(const PermDesc &d, int64_t local) {
  const int64_t tx = local % d.ntx;
  local /= d.ntx;
  const int64_t ty = local % d.nty, o = local / d.nty;
  int64_t io, oo;
  perm_outer(d, o, &io, &oo);
  const int64_t x0 = tx * d.tx, y0 = ty * d.ty;
  PermTile t;
  t.in = d.in + io + x0 * d.istr_x + y0 * d.istr_y;
  t.out = d.out + oo + x0 * d.ostr_x + y0 * d.ostr_y;
  t.cx = (int32_t)(d.nx - x0 < d.tx ? d.nx - x0 : d.tx);
  t.cy = (int32_t)(d.ny - y0 < d.ty ? d.ny - y0 : d.ty);
  return t;
}

DB_HD int32_t perm_smem_at(const PermDesc &d, int32_t x, int32_t y, int32_t b, int32_t k) {
  return d.out_major ? x * d.pitch + (y * k + b) * d.ps : y * d.pitch + (x * k + b) * d.ps;
}

template <typename T>
DB_HD void perm_tile_load(const PermDesc &d, const PermTile &t, uint8_t *sm, int tid, int nt) {
  const int32_t k = (int32_t)(d.r / d.ps);
  if (!d.out_major && d.pitch == t.cx * d.r && (t.cy == 1 || d.istr_y == d.pitch) && (t.cx == 1 || d.istr_x == d.r)) {
    perm_span(sm, t.in, (int64_t)t.cy * d.pitch, tid, nt);
    return;
  }
  const int32_t row = t.cx * k, total = t.cy * row;
  for (int32_t i = tid; i < total; i += nt) {
    const int32_t y = i / row, j = i - y * row, x = j / k, b = j - x * k;
    *reinterpret_cast<T *>(sm + perm_smem_at(d, x, y, b, k)) =
        *reinterpret_cast<const T *>(t.in + y * d.istr_y + x * d.istr_x + (int64_t)b * d.ps);
  }
}

template <typename T>
DB_HD void perm_tile_store(const PermDesc &d, const PermTile &t, const uint8_t *sm, int tid, int nt) {
  const int32_t k = (int32_t)(d.r / d.ps);
  if (d.out_major && d.pitch == t.cy * d.r && (t.cx == 1 || d.ostr_x == d.pitch) && (t.cy == 1 || d.ostr_y == d.r)) {
    perm_span(t.out, sm, (int64_t)t.cx * d.pitch, tid, nt);
    return;
  }
  const int32_t row = t.cy * k, total = t.cx * row;
  for (int32_t i = tid; i < total; i += nt) {
    const int32_t x = i / row, j = i - x * row, y = j / k, b = j - y * k;
    *reinterpret_cast<T *>(t.out + x * d.ostr_x + y * d.ostr_y + (int64_t)b * d.ps) =
        *reinterpret_cast<const T *>(sm + perm_smem_at(d, x, y, b, k));
  }
}

// ---------------------------------------------------------------------------------------------------------------- ROW
struct PermRowItem {
  int64_t row0, b0, b1;
  int32_t nrows;
};

DB_HD PermRowItem perm_row_item(const PermDesc &d, int64_t local) {
  PermRowItem it;
  if (d.segs > 1) {
    it.row0 = local / d.segs;
    it.b0 = (local - it.row0 * d.segs) * kPermTileBytes;
    it.b1 = it.b0 + kPermTileBytes < d.r ? it.b0 + kPermTileBytes : d.r;
    it.nrows = 1;
  } else {
    it.row0 = local * d.rows_per_item;
    it.nrows = (int32_t)(d.rows - it.row0 < d.rows_per_item ? d.rows - it.row0 : d.rows_per_item);
    it.b0 = 0; it.b1 = d.r;
  }
  return it;
}

// phase 1: the byte offsets of the item's rows, kept in shared memory (at most kPermTileBytes / kPermRowBytes rows)
DB_HD void perm_rows_prepare(const PermDesc &d, const PermRowItem &it, int64_t *sm, int tid, int nt) {
  for (int32_t j = tid; j < it.nrows; j += nt) perm_outer(d, it.row0 + j, &sm[2 * j], &sm[2 * j + 1]);
}

template <typename W>
DB_HD void perm_rows_copy_w(const PermDesc &d, const PermRowItem &it, const int64_t *sm, int tid, int nt) {
  const int64_t len = it.b1 - it.b0;
  // every row starts at the same offset modulo sizeof(W) on both sides (d.w divides the strides and in - out)
  int64_t h = (int64_t)((0 - (uint64_t)(uintptr_t)(d.out + it.b0)) & (sizeof(W) - 1));
  if (h > len) h = len;
  const int64_t nb = (len - h) / (int64_t)sizeof(W), tail = len - h - nb * (int64_t)sizeof(W);
  const int64_t upr = nb + h + tail, total = upr * it.nrows;
  for (int64_t i = tid; i < total; i += nt) {
    const int64_t j = i / upr, u = i - j * upr;
    const uint8_t *src = d.in + sm[2 * j] + it.b0;
    uint8_t *dst = d.out + sm[2 * j + 1] + it.b0;
    if (u < nb) {
      *reinterpret_cast<W *>(dst + h + u * (int64_t)sizeof(W)) = *reinterpret_cast<const W *>(src + h + u * (int64_t)sizeof(W));
    } else {
      const int64_t q = u - nb, off = q < h ? q : nb * (int64_t)sizeof(W) + q;
      dst[off] = src[off];
    }
  }
}

DB_HD void perm_rows_copy(const PermDesc &d, const PermRowItem &it, const int64_t *sm, int tid, int nt) {
  switch (d.w) {
    case 16: perm_rows_copy_w<PermV16>(d, it, sm, tid, nt); break;
    case 8: perm_rows_copy_w<PermV8>(d, it, sm, tid, nt); break;
    case 4: perm_rows_copy_w<uint32_t>(d, it, sm, tid, nt); break;
    case 2: perm_rows_copy_w<uint16_t>(d, it, sm, tid, nt); break;
    default: perm_rows_copy_w<uint8_t>(d, it, sm, tid, nt); break;
  }
}

// phase 1 / phase 2 of a TILE item, dispatched on the piece size
DB_HD void perm_tile_phase(const PermDesc &d, const PermTile &t, uint8_t *sm, int tid, int nt, bool store) {
  switch (d.ps) {
    case 16: store ? perm_tile_store<PermV16>(d, t, sm, tid, nt) : perm_tile_load<PermV16>(d, t, sm, tid, nt); break;
    case 8: store ? perm_tile_store<PermV8>(d, t, sm, tid, nt) : perm_tile_load<PermV8>(d, t, sm, tid, nt); break;
    case 4: store ? perm_tile_store<uint32_t>(d, t, sm, tid, nt) : perm_tile_load<uint32_t>(d, t, sm, tid, nt); break;
    case 2: store ? perm_tile_store<uint16_t>(d, t, sm, tid, nt) : perm_tile_load<uint16_t>(d, t, sm, tid, nt); break;
    default: store ? perm_tile_store<uint8_t>(d, t, sm, tid, nt) : perm_tile_load<uint8_t>(d, t, sm, tid, nt); break;
  }
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_PERMUTE_CORE_H_
