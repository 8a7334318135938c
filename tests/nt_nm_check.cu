// Host build of the sphere search of csrc/nuclear_tomo.cuh (the code the device runs).
//   nt_nm_check argsort IN OUT: IN holds 4 float64 keys per row; OUT gets argsort4's 4 int32 indices per row.
//   nt_nm_check search IN OUT: IN holds x0[3], lb[3], ub[3], r2, baseline, maxfun, maxiter, the volume's (nz, h, w) and its voxels,
//   all float64; OUT gets x[3], fun, nfev, nit, status as float64.  The objective sums the sphere as the device does.
#include <cstdio>
#include <cstring>
#include <vector>

#include "../pylinac_b200/csrc/nuclear_tomo.cuh"

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

int main(int argc, char** argv) {
    if (argc != 4) return 2;
    const std::vector<double> in = read_all(argv[2]);
    FILE* g = std::fopen(argv[3], "wb");
    if (!g) return 2;
    if (!std::strcmp(argv[1], "argsort")) {
        for (size_t r = 0; r + 4 <= in.size(); r += 4) {
            int ind[4];
            epid::nt::argsort4(&in[r], ind);
            std::fwrite(ind, sizeof(int), 4, g);
        }
    } else {
        const double* p = in.data();
        const int nz = (int)p[13], h = (int)p[14], w = (int)p[15];
        const double* vol = p + 16;
        const double r2 = p[9], baseline = p[10];
        auto func = [&](const double* x) {
            int z0, z1, y0, y1, x0, x1;
            epid::nt::sphere_span(x[2], r2, nz, z0, z1);
            epid::nt::sphere_span(x[1], r2, h, y0, y1);
            epid::nt::sphere_span(x[0], r2, w, x0, x1);
            unsigned long long s = 0;
            long long n = 0;
            for (int z = z0; z <= z1; z++)
                for (int y = y0; y <= y1; y++)
                    for (int xx = x0; xx <= x1; xx++)
                        if (epid::nt::in_sphere(xx, y, z, x[0], x[1], x[2], r2)) {
                            s += (unsigned long long)vol[((size_t)z * h + y) * w + xx];
                            n++;
                        }
            return epid::nt::contrast(s, n, baseline);
        };
        const epid::nt::Search r = epid::nt::nelder_mead(p, p + 3, p + 6, (int)p[11], (int)p[12], func);
        const double out[7] = {r.x[0], r.x[1], r.x[2], r.fun, (double)r.nfev, (double)r.nit, (double)r.status};
        std::fwrite(out, sizeof(double), 7, g);
    }
    std::fclose(g);
    return 0;
}
