// Route 0 of evk_gconv_fwd (the exact skinny-row path on evk_gemv_rows), plain C++ so that tests can compile it for the host.
#pragma once

#include "../../include/evk.h"

namespace evk {

// evk_gemv_rows stages every channel of up to 4 rows at once: R * C floats in 40 KB, R = rows rounded up to a power of 2.
// More rows are staged a channel chunk at a time.
inline bool gemv_rows_fit(int rows, int C) {
  int R = 1;
  while (R < rows) R *= 2;
  return R > 4 || (long long)R * C * 4 <= 40 * 1024;
}

// The launch is a Linear of 1..4 dense rows that the caller takes no gradient through, with what evk_gemv_rows needs.
inline bool gconv_fwd_gemv(const evk_gconv_desc* d) {
  const long long npos = (long long)d->J * d->P, rows = d->Z * npos;
  const bool dense = d->Z == 1 || (d->x_sb == npos * d->ldx && d->y_sb == npos * d->ldy);
  return d->no_grad && d->Q == 1 && d->off[0] == 0 && d->is == 1 && d->os == 1 && d->o0 == 0 && d->J <= d->Tin && d->G <= 1 &&
         d->H == 1 && !d->res && !d->in_len && !d->out_len && !(d->drop_rng && d->drop_p > 0.f) &&
         (d->act == EVK_ACT_NONE || d->act == EVK_ACT_RELU || d->act == EVK_ACT_LRELU) && rows >= 1 && rows <= 4 && d->C >= 4 &&
         d->C % 4 == 0 && d->C <= d->ldw && d->ldw % 4 == 0 && ((uintptr_t)d->w % 16) == 0 && d->ldx >= d->C && d->ldy >= d->N &&
         dense && gemv_rows_fit((int)rows, d->C);
}

}  // namespace evk
