// Host build of csrc/np_sum.cuh (the code the device runs).
//   np_sum_check IN OUT: IN holds float64 values x; for every prefix length n = 0 .. len(x), OUT gets pw(x, n) and the slot-wise
//   evaluation of block_pw for 2^9 and 2^3 threads (pw_slot, then the pairwise level combine), three float64 per n.
#include <cstdio>
#include <vector>

#include "../pylinac_b200/csrc/np_sum.cuh"

static std::vector<double> read_all(const char* path) {
    std::vector<double> v;
    FILE* f = std::fopen(path, "rb");
    if (!f) return v;
    double buf[4096];
    size_t k;
    while ((k = std::fread(buf, sizeof(double), 4096, f)) > 0) v.insert(v.end(), buf, buf + k);
    std::fclose(f);
    return v;
}

static double slots_sum(const std::vector<double>& x, long long n, int D) {
    auto at = [&](long long i) { return x[i]; };
    std::vector<double> v(1 << D);
    for (int t = 0; t < (1 << D); t++) {
        long long s, m;
        epid::np::pw_slot(n, t, D, &s, &m);
        v[t] = m < 0 ? 0.0 : epid::np::pw(at, s, m);
    }
    for (int level = D - 1; level >= 0; level--)
        for (int t = 0; t < (1 << level); t++) v[t] = v[2 * t] + v[2 * t + 1];
    return v[0];
}

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    const std::vector<double> x = read_all(argv[1]);
    FILE* g = std::fopen(argv[2], "wb");
    if (!g) return 2;
    auto at = [&](long long i) { return x[i]; };
    for (long long n = 0; n <= (long long)x.size(); n++) {
        const double out[3] = {epid::np::pw(at, 0, n), slots_sum(x, n, 9), slots_sum(x, n, 3)};
        std::fwrite(out, sizeof(double), 3, g);
    }
    std::fclose(g);
    return 0;
}
