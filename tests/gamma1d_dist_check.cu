// Host build of the segment distance of csrc/gamma1d.cuh (the routine the device runs): reads n segments (px, py, v1x, v1y, v2x,
// v2y as float64) from argv[1] and writes n distances and n python-dist values for (p, v1) and the svd flags to argv[2].
#include <cstdio>
#include <vector>

#include "../pylinac_b200/csrc/gamma1d.cuh"

int main(int argc, char** argv) {
    if (argc != 3) return 2;
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<double> in;
    double buf[6];
    while (std::fread(buf, sizeof(double), 6, f) == 6) in.insert(in.end(), buf, buf + 6);
    std::fclose(f);
    const size_t n = in.size() / 6;
    std::vector<double> out(3 * n);
    for (size_t i = 0; i < n; i++) {
        const double* s = &in[6 * i];
        bool fail = false;
        out[i] = epid::g1::segment_distance(s[0], s[1], s[2], s[3], s[4], s[5], &fail);
        out[n + i] = epid::g1::py_dist(s[0], s[1], s[2], s[3]);
        out[2 * n + i] = fail ? 1.0 : 0.0;
    }
    FILE* g = std::fopen(argv[2], "wb");
    if (!g) return 2;
    std::fwrite(out.data(), sizeof(double), out.size(), g);
    std::fclose(g);
    std::printf("%zu segments ok\n", n);
    return 0;
}
