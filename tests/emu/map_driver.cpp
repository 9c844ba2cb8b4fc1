// map_driver.cpp — TEST ONLY. Compiles the distance transform's per-column and per-row source
// (path_optimizer_2_b200/csrc/pqp_map_core.cuh) for the host and runs it in the order the two kernels of
// pqp_bounds.cu do, in place in one int32 / float buffer, so the kernel arithmetic can be checked against the
// oracle on a GPU-less box. The product has no CPU path; nothing in the package references this file.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../path_optimizer_2_b200/csrc/pqp_map_core.cuh"

// layer[rows * cols] receives the distance layer; d2[rows * cols] (optional) the squared distances
extern "C" int pqm_emu_transform(const uint8_t *img, int rows, int cols, int obstacle_max, double resolution,
                                 float *layer, int32_t *d2) {
    if (rows < 2 || cols < 2 || rows > pqm::kMaxSide || cols > pqm::kMaxSide) return 1;
    int32_t *g = reinterpret_cast<int32_t *>(layer);  // the kernels work in place in the layer
    for (int j = 0; j < cols; ++j) pqm::column_pass(img, rows, cols, j, obstacle_max, g);
    std::vector<int32_t> rg(cols), h(cols);
    std::vector<int16_t> s(cols), t(cols);
    const int32_t inf = pqm::inf_g(rows, cols);
    for (int i = 0; i < rows; ++i) {
        int32_t *row = g + (size_t)i * cols;
        std::memcpy(rg.data(), row, cols * sizeof(int32_t));
        const int n = pqm::envelope(rg.data(), cols, s.data(), t.data(), h.data());
        for (int k = 0; k < n; ++k) pqm::fill(s.data(), t.data(), h.data(), n, cols, k, rg.data());
        if (d2) std::memcpy(d2 + (size_t)i * cols, rg.data(), cols * sizeof(int32_t));
        float *out = layer + (size_t)i * cols;
        for (int u = 0; u < cols; ++u) out[u] = pqm::layer_value(rg[u], inf * inf, (float)resolution);
    }
    return 0;
}
