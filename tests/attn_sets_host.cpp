// Host harness of tests/test_attn_sets_host.py: enumerates KeySet and QuerySet (k-diffusion_b200/csrc/attn_sets.cuh, compiled here as
// plain C++) for each geometry read from stdin as "type h w param shift" lines.  Writes int32 records to stdout, per geometry:
//   T, KeySet::count(), QuerySet::max_count();
//   T rows of KeySet::count() entries: row q holds token(j) of query q's key set (-1 = masked);
//   T rows of T + 1 entries: row k holds QuerySet::count() of key k, then its token(t) (-1 = masked), padded with -2.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "attn_sets.cuh"

int main() {
  int type, h, w, param, shift;
  std::vector<int32_t> buf;
  while (std::scanf("%d %d %d %d %d", &type, &h, &w, &param, &shift) == 5) {
    const int T = h * w, nk = kdb::KeySet::count(type, h, w, param), maxq = kdb::QuerySet::max_count(type, h, w, param);
    buf.assign({T, nk, maxq});
    for (int q = 0; q < T; ++q) {
      kdb::KeySet ks{};
      ks.init(type, h, w, param, shift, q);
      for (int j = 0; j < ks.count(); ++j) buf.push_back(ks.token(j));
    }
    for (int k = 0; k < T; ++k) {
      kdb::QuerySet qs{};
      qs.init(type, h, w, param, shift, k);
      const int nq = qs.count();
      buf.push_back(nq);
      for (int t = 0; t < T; ++t) buf.push_back(t < nq ? qs.token(t) : -2);
    }
    std::fwrite(buf.data(), sizeof(int32_t), buf.size(), stdout);
  }
  return 0;
}
