// ref_knn_harness.cpp -- a C entry point around the reference's own third-party headers, built by
// oracle/build_ref_knn.py into oracle/_ref/libref_knn.so (test and benchmark infrastructure only):
//   ref_knn_mean_dist  the query of compute_mean_neighbor_distances (src/core/splat_data.cpp:63-111): a nanoflann
//                      KDTreeSingleIndexAdaptor over L2_Simple_Adaptor<float>, leaf size 10, KNNResultSet(min(4, N)),
//                      SearchParameters(10) (eps = 10: approximate), the first three distances above 1e-8 averaged;
//                      OpenMP over the queries above 1000 points, as in the reference
//   ref_write_ply      write_ply_impl (splat_data.cpp:113-169): one float32 vertex property group per array, in the
//                      given order, written by tinyply as binary little-endian
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <fstream>
#include <string>
#include <vector>

#include "nanoflann.hpp"
#define TINYPLY_IMPLEMENTATION
#include "tinyply.hpp"

namespace {

struct Cloud {
    const float *p;
    size_t n;
    size_t kdtree_get_point_count() const { return n; }
    float kdtree_get_pt(size_t i, size_t d) const { return p[i * 3 + d]; }
    template <class B> bool kdtree_get_bbox(B &) const { return false; }
};

using Tree = nanoflann::KDTreeSingleIndexAdaptor<nanoflann::L2_Simple_Adaptor<float, Cloud>, Cloud, 3>;

} // namespace

extern "C" int ref_knn_mean_dist(const float *pts, int n, float *out) {
    if (n <= 1) {
        for (int i = 0; i < n; ++i) out[i] = 0.01f;
        return 0;
    }
    Cloud cloud{pts, (size_t)n};
    Tree tree(3, cloud, nanoflann::KDTreeSingleIndexAdaptorParams(10));
    tree.buildIndex();
#pragma omp parallel for if (n > 1000)
    for (int i = 0; i < n; ++i) {
        const float q[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        const size_t k = std::min(4, n);
        std::vector<size_t> idx(k);
        std::vector<float> d2(k);
        nanoflann::KNNResultSet<float> rs(k);
        rs.init(idx.data(), d2.data());
        tree.findNeighbors(rs, q, nanoflann::SearchParameters(10));
        float sum = 0.0f;
        int valid = 0;
        for (size_t j = 0; j < k && valid < 3; ++j)
            if (d2[j] > 1e-8f) {
                sum += std::sqrt(d2[j]);
                ++valid;
            }
        out[i] = valid > 0 ? sum / valid : 0.01f;
    }
    return 0;
}

// groups: n_groups arrays of rows x cols[g] floats; names: every column's property name, '\n'-separated
extern "C" int ref_write_ply(const char *path, size_t rows, int n_groups, const float *const *groups, const int *cols,
                             const char *names) {
    std::vector<std::string> all;
    std::string cur;
    for (const char *c = names; *c; ++c) {
        if (*c == '\n') {
            all.push_back(cur);
            cur.clear();
        } else {
            cur += *c;
        }
    }
    if (!cur.empty()) all.push_back(cur);
    tinyply::PlyFile ply;
    size_t off = 0;
    for (int g = 0; g < n_groups; ++g) {
        if (off + cols[g] > all.size()) return -1;
        std::vector<std::string> attrs(all.begin() + off, all.begin() + off + cols[g]);
        ply.add_properties_to_element("vertex", attrs, tinyply::Type::FLOAT32, rows,
                                      reinterpret_cast<uint8_t *>(const_cast<float *>(groups[g])),
                                      tinyply::Type::INVALID, 0);
        off += cols[g];
    }
    std::filebuf fb;
    if (!fb.open(path, std::ios::out | std::ios::binary)) return -2;
    std::ostream os(&fb);
    ply.write(os, true);
    return 0;
}
