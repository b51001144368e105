// Polyphase plan of a conv's data gradient (evk_gconv_dgrad), plain C++ so that tests can compile it for the host.
//
// The forward reads input row u = j*is + off[q] for output j and tap q, so
//   dX[u] = sum over (j, q) with j*is + off[q] == u of dY[j] W[q].
// For is == 1 every tap reaches every u: one phase, a stride-1 tap sum over dY with offsets -off[q].  For is > 1 the taps
// must sit at consecutive offsets (off[q] = off[0] + q, dilation 1); then tap q only reaches the u with u = off[q] (mod is),
// and the taps of one residue rho = q mod is fill every is-th row of dX as a stride-1 tap sum over dY.
#pragma once

#include "../../include/evk.h"

namespace evk {

// One stride-1 launch of the plan: rows u = u0 + is*jj of dX, jj < J, sum taps q0, q0 + is, ... (nq of them); tap k of the
// phase reads dY row jj + off[k].
struct DgradPhase {
  int u0, J, q0, nq;
  int off[EVK_MAX_TAPS];
};

// The phase of tap residue rho (0 <= rho < is) of a conv with Q taps at offsets off[], stride is and Tin rows of dX.
// False when no tap or no row of dX has that residue.
inline bool dgrad_phase(const int* off, int Q, int is, int Tin, int rho, DgradPhase& ph) {
  if (rho >= Q) return false;
  ph.u0 = (off[rho] % is + is) % is;
  if (ph.u0 >= Tin) return false;
  ph.q0 = rho;
  ph.nq = (Q - rho + is - 1) / is;
  ph.J = (Tin - ph.u0 + is - 1) / is;
  for (int k = 0; k < ph.nq; ++k) ph.off[k] = (ph.u0 - off[rho + k * is]) / is;     // an exact division
  return true;
}

}  // namespace evk
