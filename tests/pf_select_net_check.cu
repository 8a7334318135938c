// Host check of the pruned selection networks of pf_win_common.cuh (compiled and run by tests/test_pf_select_net.py).
// Every list is evaluated exactly as the device applies it (a NET_MIN comparator writes only its minimum wire, a NET_MAX one only
// its maximum wire) and its output wires are compared with the order statistics of the input:
//   exhaustively over all 2^n 0/1 inputs for n <= 20 (0/1 principle: min / max commute with every threshold), 64 inputs per word;
//   on random inputs with many ties for every n (10^5 per exact network, 2 x 10^4 per key count of a padded one).
// Checked uses: pair_median_exact<N> (wires (N-1)/2, N/2) and rank_keys<N> (nr <= N keys behind which ceil(p/2) zero and
// floor(p/2) all-ones slots are padded, p = N - nr; the middles of the keys on wires N/2 - 1, N/2).
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <random>
#include <utility>
#include <vector>

#include "../pylinac_b200/csrc/pf_win_common.cuh"

using epid::NetList;

static int g_fail = 0;

template <class T, class Min, class Max>
static void apply(const NetList& L, T* r, Min mn, Max mx) {
    for (int i = 0; i < L.n; i++) {
        const T a = r[L.a[i]], b = r[L.b[i]];
        if (L.k[i] != epid::NET_MAX) r[L.a[i]] = mn(a, b);
        if (L.k[i] != epid::NET_MIN) r[L.b[i]] = mx(a, b);
    }
}

// wires: N; the nr data values sit on wires 0..nr-1, then zeros up to zeros_end, then all-ones; checks wires o1, o2 against
// the data's order statistics (nr - 1) / 2 and nr / 2 (the pair median: o1 == o2 for odd nr)
static void check(const NetList& L, int N, int nr, int o1, int o2, const char* what, int trials, std::mt19937_64& rng) {
    const int zeros_end = nr + (N - nr + 1) / 2;
    // 0/1 inputs, 64 at a time: bit j of word w is input vector (base + j)
    if (nr <= 20) {
        const uint64_t total = 1ull << nr;
        for (uint64_t base = 0; base < total; base += 64) {
            std::vector<uint64_t> r(N);
            for (int w = 0; w < N; w++) {
                uint64_t bits = w < zeros_end ? 0ull : ~0ull;
                if (w < nr && w < 6) {
                    bits = 0;
                    for (int j = 0; j < 64; j++) bits |= (uint64_t)((j >> w) & 1) << j;
                } else if (w < nr) {
                    bits = ((base >> w) & 1) ? ~0ull : 0ull;
                }
                r[w] = bits;
            }
            apply(L, r.data(), [](uint64_t a, uint64_t b) { return a & b; }, [](uint64_t a, uint64_t b) { return a | b; });
            const int nj = total - base < 64 ? (int)(total - base) : 64;
            for (int j = 0; j < nj; j++) {
                const uint64_t v = base + j;
                const int ones = __builtin_popcountll(v);
                // sorted 0/1 data: position q holds 1 iff q >= nr - ones
                const int e1 = (nr - 1) / 2 >= nr - ones, e2 = nr / 2 >= nr - ones;
                if ((int)((r[o1] >> j) & 1) != e1 || (int)((r[o2] >> j) & 1) != e2) {
                    if (g_fail++ < 10) printf("FAIL %s N=%d nr=%d 0/1 input %llx\n", what, N, nr, (unsigned long long)v);
                    return;
                }
            }
        }
    }
    // random inputs with ties (value ranges 2, 3, 16, 65536 and the full 64 bits, so the pads tie with data too)
    const uint64_t ranges[5] = {2, 3, 16, 65536, 0};
    std::vector<uint64_t> r(N), d(nr);
    for (int t = 0; t < trials; t++) {
        const uint64_t R = ranges[t % 5];
        for (int i = 0; i < nr; i++) {
            uint64_t v = R ? rng() % R : rng();
            if (R == 3) v = v == 2 ? ~0ull : v;        // data equal to the all-ones pad
            d[i] = v;
        }
        for (int w = 0; w < N; w++) r[w] = w < nr ? d[w] : (w < zeros_end ? 0ull : ~0ull);
        apply(L, r.data(), [](uint64_t a, uint64_t b) { return a < b ? a : b; }, [](uint64_t a, uint64_t b) { return a < b ? b : a; });
        std::sort(d.begin(), d.end());
        if (r[o1] != d[(nr - 1) / 2] || r[o2] != d[nr / 2]) {
            if (g_fail++ < 10) printf("FAIL %s N=%d nr=%d random trial %d\n", what, N, nr, t);
            return;
        }
    }
}

// pair_median_exact<N>: all N wires hold data
template <int N>
static void check_exact(std::mt19937_64& rng) {
    check(epid::SelectNet<N, (N - 1) / 2, N / 2>::L, N, N, (N - 1) / 2, N / 2, "exact", 100000, rng);
}
template <int... I>
static void check_exact_all(std::integer_sequence<int, I...>, std::mt19937_64& rng) {
    (check_exact<I + 1>(rng), ...);
}

// symmetric padding: the device reads wire N/2 for both middles when nr is odd
template <int N>
static void check_padded(const char* what, std::mt19937_64& rng) {
    const NetList& L = epid::SelectNet<N, N / 2 - 1, N / 2>::L;
    for (int nr = 1; nr <= N; nr++) check(L, N, nr, (nr & 1) ? N / 2 : N / 2 - 1, N / 2, what, 20000, rng);
}

int main() {
    std::mt19937_64 rng(12345);
    check_exact_all(std::make_integer_sequence<int, 32>{}, rng);
    check_padded<16>("rank_keys<16>", rng);
    check_padded<32>("rank_keys<32>", rng);
    // sizes of the pruned lists against the sorting networks (comparators: both outputs + one output)
    const int ns[] = {6, 12, 13, 16, 26, 32};
    for (int N : ns) {
        const NetList full = epid::batcher_net(N);
        const NetList sel = epid::prune_net(full, (1ull << ((N - 1) / 2)) | (1ull << (N / 2)));
        int half = 0;
        for (int i = 0; i < sel.n; i++) half += sel.k[i] != epid::NET_BOTH;
        printf("N=%d sort %d comparators, median %d + %d half\n", N, full.n, sel.n - half, half);
    }
    if (g_fail) { printf("%d failures\n", g_fail); return 1; }
    printf("ok\n");
    return 0;
}
