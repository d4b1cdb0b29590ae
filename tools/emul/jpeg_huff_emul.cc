// tools/emul/jpeg_huff_emul.cc -- TEST INFRASTRUCTURE.  Runs the table builder and the step rule of the JPEG entropy passes on the host.
//
// huff_sync_intra, huff_sync_walk and huff_write (dali_b200/csrc/jpeg.cu) look up an entry of the tables BuildDeviceTable makes and take
// the step huff_step picks (dali_b200/csrc/jpeg_huff_core.h).  This file compiles those with the host compiler and restates the
// passes' symbol loop around them, so that tests/test_jpeg_huff_core_cpu.py can check every entry against a plain one-symbol decoder,
// and whole streams decoded with pairs against the same streams decoded one symbol per step, on a machine without a GPU.
//   g++ -std=c++17 -O2 -shared -fPIC tools/emul/jpeg_huff_emul.cc
#include "../../dali_b200/csrc/jpeg_huff_core.h"

using namespace dalib200;

namespace {

// slow_lookup (jpeg.cu) with the canonical search only: the direct long-code table holds the same codes
uint32_t slow_entry(const HuffSlow &sl, uint32_t hi, bool is_dc) {
  const int32_t code16 = (int32_t)(hi >> 16);
  uint32_t len = (is_dc ? kDcLutBits : kAcLutBits) + 1, sym = 0;
  while (len <= 16 && code16 >= sl.maxcode[len]) len++;
  if (len > 16) len = 17;
  else sym = sl.vals[(sl.valoff[len] + (code16 >> (16 - len))) & 0xFF];
  return huff_entry(len, sym, is_dc);
}

// the 32 bits of the stream at bit `pos`, MSB first; bits behind the stream read as 0
uint32_t peek32(const uint8_t *d, uint32_t nbytes, uint32_t pos) {
  uint64_t w = 0;
  for (uint32_t k = 0; k < 5; k++) {
    const uint32_t b = (pos >> 3) + k;
    w = (w << 8) | (b < nbytes ? d[b] : 0u);
  }
  return (uint32_t)(w >> (8 - (pos & 7)));
}

// huff_write's coefficient stores of a step taken at window `hi` in block position z (AC): the first symbol of a pair (when it has a
// value) at z + adv1 - 1, the step's last symbol at min(z + adv - 1, 63).  out = (zig-zag index, value) x 2, index -1 = no store.
void ac_stores(uint32_t e, uint32_t st, uint32_t hi, uint32_t z, int32_t *out) {
  const uint32_t one = e >> 16, tb = step_bits(st), s = step_size(st), tb1 = step_bits(one), s1 = step_size(one);
  out[0] = out[2] = -1; out[1] = out[3] = 0;
  if (tb != tb1 && s1) { out[0] = (int32_t)(z + step_adv(one) - 1u); out[1] = huff_extend(hi, tb1, s1); }
  if (s) { const uint32_t zz = z + step_adv(st) - 1u; out[2] = (int32_t)(zz < 63u ? zz : 63u); out[3] = huff_extend(hi, tb, s); }
}

}  // namespace

// bits[1..16] (bits[0] unused), vals[256]: one DHT table; lut gets 1 << kDcLutBits or 1 << kAcLutBits entries
extern "C" void emul_build(const uint8_t *bits, const uint8_t *vals, int is_dc, uint32_t *lut) {
  HuffSlow slow;
  BuildDeviceTable(bits, vals, lut, slow, is_dc != 0);
}

// One AC step per query i, from bit 0 of window hi[i] at zig-zag position z[i] with room_pos[i] bits to the limit.  out[8 i ..]:
// bits consumed, zig-zag advance, the two stores of ac_stores; entry 0 (a code behind the first level) gives bits consumed 0.
extern "C" void emul_steps(const uint32_t *lut, int n, const uint32_t *hi, const int32_t *z, const uint32_t *room_pos, int32_t *out) {
  for (int i = 0; i < n; i++) {
    int32_t *o = out + 8 * i;
    const uint32_t e = lut[hi[i] >> (32 - kAcLutBits)];
    o[0] = o[1] = 0; o[2] = o[4] = -1; o[3] = o[5] = 0;
    if (e == 0) continue;
    const uint32_t st = huff_step(e, pair_threshold(z[i], 0u, room_pos[i]));
    o[0] = (int32_t)step_bits(st);
    o[1] = (int32_t)step_adv(st);
    ac_stores(e, st, hi[i], (uint32_t)z[i], o + 2);
  }
}

// decode_span / huff_write's loop over the symbols of `data` that start in [pos, end), from block position (c, z), with one symbol
// per step (pairs == 0) or with huff_step.  tables: bits[4][17] and vals[4][256] for DC0 DC1 AC0 AC1; tsel[c] = dc table | ac table
// << 8 of block c of the MCU.  state = (pos, c, z, nb, steps): nb counts the blocks completed in the stream, steps the lookups (both
// carried from span to span); block nb's coefficients (DC in slot 0, as decoded, AC at their zig-zag index) go to coef[64 * nb] while
// nb < max_blocks.
extern "C" void emul_decode(const uint8_t *data, uint32_t nbytes, const uint8_t *bits, const uint8_t *vals, const int32_t *tsel, int bpm,
                            uint32_t *state, int pairs, uint32_t end, int16_t *coef, int max_blocks) {
  static uint32_t lut[kLutWords];
  HuffSlow slow[4];
  for (int t = 0; t < 4; t++) BuildDeviceTable(bits + 17 * t, vals + 256 * t, lut + LutOffset(t), slow[t], t < 2);
  uint32_t pos = state[0], nb = state[3], steps = state[4];
  int c = (int)state[1], z = (int)state[2];
  while (pos < end) {
    const int td = tsel[c] & 255, ta = tsel[c] >> 8;
    const uint32_t hi = peek32(data, nbytes, pos);
    const bool is_dc = z == 0;
    uint32_t e = is_dc ? lut[LutOffset(td) + (hi >> (32 - kDcLutBits))] : lut[LutOffset(2 + ta) + (hi >> (32 - kAcLutBits))];
    if (e == 0) e = slow_entry(slow[is_dc ? td : 2 + ta], hi, is_dc);
    const uint32_t st = pairs ? huff_step(e, pair_threshold(z, pos, end)) : e >> 16;
    const int b = (int)nb;
    if (b < max_blocks) {
      if (is_dc) {
        coef[64 * b] = (int16_t)huff_extend(hi, step_bits(st), step_size(st));
      } else {
        int32_t o[4];
        ac_stores(e, st, hi, (uint32_t)z, o);
        if (o[0] >= 0) coef[64 * b + o[0]] = (int16_t)o[1];
        if (o[2] >= 0) coef[64 * b + o[2]] = (int16_t)o[3];
      }
    }
    pos += step_bits(st);
    z += (int)step_adv(st);
    steps++;
    if (z >= 64) { z = 0; c = c + 1 == bpm ? 0 : c + 1; nb++; }
  }
  state[0] = pos; state[1] = (uint32_t)c; state[2] = (uint32_t)z; state[3] = nb; state[4] = steps;
}
