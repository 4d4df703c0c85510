// K2t instantiations: team walk for the LPV = 8 row shapes.
#include "team_impl.cuh"

namespace ehb {

// Vector-load steps (4 vectors each) a team warp keeps in flight: the U template argument of K2t.  Registers of
// loads in flight per lane are sized so that 7 CTAs fit an SM (T = 2: 64, T = 3 and 4: 32), except that T = 4
// keeps the full 16-vector batches when the batch is so small that registers are no constraint (<= 3 CTAs of 128
// threads per SM of the H100's 132 at ~125 registers).
constexpr uint32_t kTeamWideMaxQueries = 132u * 3u;
__host__ __device__ constexpr int team_u_wide(int NQ) { return NQ <= 2 ? 8 : (NQ <= 4 ? 4 : 2); }
__host__ __device__ constexpr int team_u_narrow(int NQ) { return NQ <= 2 ? 4 : (NQ <= 4 ? 2 : 1); }
static bool team_wide(uint32_t T, uint32_t nq) { return T == 2 || (T >= 4 && nq <= kTeamWideMaxQueries); }

uint32_t team_eval_steps(uint32_t T, uint32_t dpad, uint32_t nq) {
  const int NQ = (int)(dpad / 32u);
  return (uint32_t)(team_wide(T, nq) ? team_u_wide(NQ) : team_u_narrow(NQ));
}

template <int NQ, int T, int U>
static cudaError_t team_kpl(const GraphView& g, uint32_t hash_size, const float* queries, uint32_t nq, uint32_t k,
                            uint32_t ef, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                            uint32_t* stats, cudaStream_t s) {
  if (ef <= 64) return launch_team_t<NQ, 2, T, U>(g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
  if (ef <= 128) return launch_team_t<NQ, 4, T, U>(g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
  return launch_team_t<NQ, 8, T, U>(g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
}

template <int NQ>
static cudaError_t team_t(uint32_t T, const GraphView& g, uint32_t hash_size, const float* queries, uint32_t nq,
                          uint32_t k, uint32_t ef, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                          uint32_t* stats, cudaStream_t s) {
  constexpr int U2 = team_u_wide(NQ), U4 = team_u_narrow(NQ);
  if (T >= 4 && team_wide(T, nq))
    return team_kpl<NQ, 4, U2>(g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
  if (T >= 4) return team_kpl<NQ, 4, U4>(g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
  if (T == 3) return team_kpl<NQ, 3, U4>(g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
  return team_kpl<NQ, 2, U2>(g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
}

// ef <= 256, dpad in {32, 64, 128, 256}
cudaError_t launch_search_team(uint32_t T, const GraphView& g, uint32_t hash_size, const float* queries, uint32_t nq,
                               uint32_t k, uint32_t ef, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                               uint32_t* stats, cudaStream_t s) {
  if (nq == 0) return cudaSuccess;
  switch (g.dpad) {
    case 32: return team_t<1>(T, g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    case 64: return team_t<2>(T, g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    case 128: return team_t<4>(T, g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    case 256: return team_t<8>(T, g, hash_size, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace ehb
