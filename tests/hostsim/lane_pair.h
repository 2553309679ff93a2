// lane_pair.h — TEST INFRASTRUCTURE (tests/hostsim): the physics and epilogue of the lane-pair step
// (step_env_kernel<W, P, 2> in csrc/spec_kernel.cuh) run on the CPU.  The two lanes of an env's pair run one
// after the other between exchange points; each shuffle becomes "both lanes have evaluated, hand each lane the
// other's value".  Same device functions as the kernel: rounds, sums in item order, split stores.  The kernel's
// prologue (action ingest, broad phase) is not restated here.  Not product code.
#pragma once
#include <type_traits>

namespace vmas {

template <class W, class P>
void pair_env_step(const SpecArgs& a, const long env, const uint32_t* mask_words, const EpiArgs* epi) {
  constexpr int E = W::E, NA = W::A;
  using R = SpecRounds<W, 2>;
  SpecRows<W> rows[2];
  EnvRegs<E> r[2];
  float afx[2][NA > 0 ? NA : 1], afy[2][NA > 0 ? NA : 1], atq[2][NA > 0 ? NA : 1];
  for (int g = 0; g < 2; ++g) {
    rows[g].load_pos_rot(a, env);
    rows[g].load_rest(a, env);
    rows[g].unpack_pos_rot(r[g]);
    rows[g].unpack_rest(r[g], afx[g], afy[g], atq[g]);
  }
  for (int sub = a.first_substep; sub < a.first_substep + a.n_substeps; ++sub) {
    static_for<(spec_n_trig<W>() + 1) / 2>([&](auto ki) {
      constexpr int K = decltype(ki)::value;
      float s[2], c[2];
      for (int g = 0; g < 2; ++g) spec_trig_round_eval<W, 2, K>(r[g], g == 1, s[g], c[g]);
      for (int g = 0; g < 2; ++g) spec_trig_round_put<W, 2, K>(r[g], g == 1, s[g], c[g], s[1 - g], c[1 - g]);
    });
    for (int g = 0; g < 2; ++g) spec_entity_forces<W>(r[g], afx[g], afy[g], atq[g]);
    static_for<R::N>([&](auto ki) {
      constexpr int K = decltype(ki)::value;
      if constexpr (R::template I0<K> == R::template I1<K>) {
        uint32_t sig = 0;
        for (int g = 0; g < 2; ++g) spec_item<W, R::template I0<K>, false>(r[g], a, env, mask_words, sig);
      } else {
        ItemOut o[2];
        for (int g = 0; g < 2; ++g) o[g] = spec_round_eval<W, 2, K>(r[g], a, env, mask_words, g == 1);
        for (int g = 0; g < 2; ++g) spec_round_add<W, 2, K>(r[g], a, mask_words, o[g], o[1 - g], g == 1);
      }
    });
    for (int g = 0; g < 2; ++g) spec_integrate<W>(r[g], sub);
  }
  for (int g = 0; g < 2; ++g) rows[g].store(a, env, r[g], afx[g], afy[g], atq[g], 2, g);
  if constexpr (!std::is_void_v<P>) {
    if (a.first_substep + a.n_substeps == W::cfg.substeps)
    {
      float carry[8];  // lane 0's reads of the shaping carries, in program order, for lane 1 (the shuffle)
      int n0 = 0, n1 = 0;
      spec_epilogue<W, P>(r[0], a, *epi, env, 2, 0, [&](float v) { return carry[n0++] = v; });
      spec_epilogue<W, P>(r[1], a, *epi, env, 2, 1, [&](float) { return carry[n1++]; });
    }
  }
}

}  // namespace vmas
