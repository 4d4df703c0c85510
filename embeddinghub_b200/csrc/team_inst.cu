// K2t instantiations: team walk for the LPV = 8 row shapes.
#include "team_impl.cuh"

namespace ehb {

template <int NQ, int T, int U>
static cudaError_t team_kpl(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                            uint32_t ef, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                            uint32_t* stats, cudaStream_t s) {
  const uint32_t hs = p.cfg.hash_size;
  switch (p.kpl) {
    case 2: return launch_team_t<NQ, 2, T, U>(g, hs, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    case 4: return launch_team_t<NQ, 4, T, U>(g, hs, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    case 8: return launch_team_t<NQ, 8, T, U>(g, hs, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_search_team(const WalkPlan& p, const GraphView& g, const float* queries, uint32_t nq, uint32_t k,
                               uint32_t ef, uint64_t* out_labels, float* out_dists, uint32_t* out_counts,
                               uint32_t* stats, cudaStream_t s) {
  if (nq == 0) return cudaSuccess;
  if (p.form != WalkForm::team || p.bf16 || p.lpv != 8) return cudaErrorInvalidValue;
  return with_dpad<256>(g.dpad, [&](auto d) {
    constexpr int NQ = row_nq(decltype(d)::value, decltype(d)::value * 4u);
    constexpr uint32_t UW = eval_u(NQ, 1), UN = eval_u(NQ, 2);  // wide and narrow U
    // the (T, U) pairs ehb_index::walk_plan chooses: T = 2 and 4 with the wide U, T = 3 and 4 with the narrow one
    const uint32_t T = p.T, U = p.U;
    if (T == 2 && U == UW) return team_kpl<NQ, 2, UW>(p, g, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    if (T == 3 && U == UN) return team_kpl<NQ, 3, UN>(p, g, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    if (T == 4 && U == UW) return team_kpl<NQ, 4, UW>(p, g, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    if (T == 4 && U == UN) return team_kpl<NQ, 4, UN>(p, g, queries, nq, k, ef, out_labels, out_dists, out_counts, stats, s);
    return cudaErrorInvalidValue;
  });
}

}  // namespace ehb
