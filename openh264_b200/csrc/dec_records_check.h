// dec_records_check.h — the argument check of the construct stage's test hooks: b2h264_debug_decode_records (enc_kernels.cu) and its
// host-build twin emu_decode_records (tests/emu/decode_records_hooks.cu) refuse the same arguments.  Host code; include after
// dec_mb.cuh.  True when n streams of mb_w x mb_h records (stream-major), their chroma QP offsets and n_refs reference slots fit
// what dec_one_mb reads: a geometry of 1..512 macroblocks a side, 1..16 slots, offsets in -12..12, QPs up to 51, known types and
// sub-partitions, availability bits only towards macroblocks inside the picture, the reference slot of every list a
// macroblock uses inside 0..n_refs - 1, and list-1 records wherever a B record needs them.
#pragma once

namespace mbk {

inline bool dec_records_ok(int n, int mb_w, int mb_h, const int* cqp_off, const MbOut* recs, const DecMbAux* aux, const DecMbAuxB* aux_b,
                           int n_refs, const uint8_t* refs, const uint8_t* planes, const MbInfo* mbi) {
  if (n < 1 || mb_w < 1 || mb_h < 1 || mb_w > 512 || mb_h > 512 || n_refs < 1 || n_refs > 16 || !cqp_off || !recs || !aux || !refs ||
      !planes || !mbi)
    return false;
  const int n_mb = mb_w * mb_h;
  for (int s = 0; s < n; s++) {
    if (cqp_off[s] < -12 || cqp_off[s] > 12) return false;
    for (int i = 0; i < n_mb; i++) {
      const MbOut& m = recs[(size_t)s * n_mb + i];
      const DecMbAux& a = aux[(size_t)s * n_mb + i];
      const int x = i % mb_w, y = i / mb_w;
      const int geo = (x > 0 ? NB_LEFT : 0) | (y > 0 ? NB_TOP : 0) | (x > 0 && y > 0 ? NB_TOPLEFT : 0) | (y > 0 && x < mb_w - 1 ? NB_TOPRIGHT : 0);
      if (m.mb_type > MBT_BSKIP || m.qp > 51 || (a.avail & ~geo)) return false;
      for (int k = 0; k < 4; k++) {
        if (a.sub_type[k] > 3) return false;
        if (MBT_IS_B(m.mb_type)) {
          if (!aux_b) return false;
          const DecMbAuxB& b = aux_b[(size_t)s * n_mb + i];
          if (((b.pred[k] & DECB_L0) && (a.ref_idx[k] < 0 || a.ref_idx[k] >= n_refs)) ||
              ((b.pred[k] & DECB_L1) && (b.ref_idx[k] < 0 || b.ref_idx[k] >= n_refs)))
            return false;
        } else if (MBT_IS_INTER(m.mb_type) && (a.ref_idx[k] < 0 || a.ref_idx[k] >= n_refs)) {
          return false;
        }
      }
    }
  }
  return true;
}

}  // namespace mbk
