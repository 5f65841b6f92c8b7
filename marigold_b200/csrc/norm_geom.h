// Thread geometry of the GroupNorm kernel (norm.cu).
#pragma once

namespace mgb {

constexpr int kGnThreads = 256;
constexpr int kGnLoads = 8;          // float4 loads in flight per thread and round
constexpr int kGnMaxChunks = 1056;   // CTAs per image (8 per SM of an H100 SXM)

// Thread geometry: Tq lanes along channel quads x Tp lanes along pixels; a thread owns Kq quads (Kq in {1, 2, 4}) and
// R = 8 / Kq pixels per round, so that ALL of a round's loads are issued before anything is consumed. These kernels
// run between two GEMMs on tensors that mostly sit in L2: they are bound by dependent load latency, not bandwidth
// (walking pixels with 2-3 dependent round trips per quad would serialise them).
struct GnGeom {
  int Q;          // C / 4
  int Tq, Tp;     // Tq * Tp <= 256
  int Kq, R;      // quads per thread, pixels per thread and round (Kq * R == kGnLoads)
  int chunks, P;  // pixel chunks per image, pixels per chunk (a multiple of Tp * R)
};

static inline bool gn_geometry(int HW, int C, GnGeom* g, int max_chunks = kGnMaxChunks) {
  if (C % 4) return false;
  g->Q = C / 4;
  int best = -1;
  for (int kq = 1; kq <= 4; kq *= 2) {
    if (g->Q % kq) continue;
    const int tq = g->Q / kq;
    if (tq > kGnThreads) continue;
    const int tp = kGnThreads / tq;
    if (tq * tp > best) { best = tq * tp; g->Tq = tq; g->Tp = tp; g->Kq = kq; }
  }
  if (best < 0) return false;
  g->R = kGnLoads / g->Kq;
  const int per_round = g->Tp * g->R;
  long long rounds_total = (HW + per_round - 1) / per_round;
  long long rounds = (rounds_total + max_chunks - 1) / max_chunks;
  g->P = int(rounds) * per_round;
  g->chunks = (HW + g->P - 1) / g->P;
  return true;
}

}  // namespace mgb
