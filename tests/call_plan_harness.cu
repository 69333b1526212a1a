// Test-only harness: the host side of a forward call's plan (pointdsc_b200/csrc/sets.cuh, the header the engine compiles):
// set_sizes, attn_key_split, attn_call_splits, plan_call and attn_partial_items.  tests/test_call_plan_host.py compiles it with
// the engine's nvcc flags and calls it through ctypes.  It makes no CUDA call, so it runs without a GPU.
#include "sets.cuh"

// out[9 i ..]: S, k, QT, KT, NS, sc_rowmajor, sc_tiled, dist, knn of a set of Ns[i] rows
extern "C" void plan_set_sizes(const int* Ns, int n, double ratio, int k_cfg, long long* out) {
  for (int i = 0; i < n; ++i) {
    const pdsc::SetSizes z = pdsc::set_sizes(Ns[i], ratio, k_cfg);
    const long long v[9] = {z.S, z.k, z.QT, z.KT, z.NS, z.sc_rowmajor, z.sc_tiled, z.dist, z.knn};
    for (int j = 0; j < 9; ++j) out[9 * i + j] = v[j];
  }
}

// out[2 i ..]: sp, TS of a set of Ns[i] rows in a call that runs split
extern "C" void plan_key_split(const int* Ns, int n, int invariant, int num_sms, int* out) {
  for (int i = 0; i < n; ++i) pdsc::attn_key_split(Ns[i], invariant, num_sms, &out[2 * i], &out[2 * i + 1]);
}

extern "C" int plan_call_splits(long long qtiles, long long items, int num_sms, int invariant) {
  return pdsc::attn_call_splits(qtiles, items, num_sms, invariant) ? 1 : 0;
}

// out: B, N, S, k, k_min, R, sc_rowmajor, sc_tiled, seeds, dist, knn, qtiles, ktiles, attn_items, attn_split, attn_invariant,
// num_sms, attn_partial_items of the call (offsets == nullptr: B sets of N_uniform rows)
extern "C" void plan_call(int B, int N_uniform, const int32_t* offsets, double ratio, int k_cfg, int tc, int invariant,
                          int num_sms, long long* out) {
  const pdsc::CallShape s = pdsc::plan_call(B, N_uniform, offsets, ratio, k_cfg, tc != 0, invariant, num_sms);
  const long long v[18] = {s.B, s.N, s.S, s.k, s.k_min, (long long)s.R, (long long)s.sc_rowmajor, (long long)s.sc_tiled,
                           (long long)s.seeds, (long long)s.dist, (long long)s.knn, s.qtiles, s.ktiles, s.attn_items,
                           s.attn_split, s.attn_invariant, s.num_sms, (long long)pdsc::attn_partial_items(s)};
  for (int j = 0; j < 18; ++j) out[j] = v[j];
}
