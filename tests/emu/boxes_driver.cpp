// boxes_driver.cpp — TEST ONLY. Compiles the obstacle-box stamping and the distance transform's source
// (path_optimizer_2_b200/csrc/pqp_map_core.cuh) for the host and runs them in the order the box instantiation of the
// column kernel and the row kernel of pqp_bounds.cu do: base image into g, each box stamped column by column (the same
// bounding-box row range and predicate, without the per-block culling, which only skips boxes), the column sweeps, the
// row pass. The product has no CPU path; nothing in the package references this file.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../path_optimizer_2_b200/csrc/pqp_map_core.cuh"

// boxes [k][5] in the frame of a map centred at (cx, cy); layer[rows * cols] receives the distance layer, d2 (optional)
// the squared distances
extern "C" int pqm_emu_boxes_transform(const uint8_t *img, int rows, int cols, int obstacle_max, double resolution,
                                       double cx, double cy, const double *boxes, int k, float *layer, int32_t *d2) {
    if (rows < 2 || cols < 2 || rows > pqm::kMaxSide || cols > pqm::kMaxSide || k < 0) return 1;
    const pqm::Cells m{rows, cols, resolution, 0.5 * rows * resolution, 0.5 * cols * resolution, cx, cy};
    const double ms = pqm::map_slack(m);
    int32_t *g = reinterpret_cast<int32_t *>(layer);  // the kernels work in place in the layer
    std::vector<pqm::Box> live;
    for (int b = 0; b < k; ++b) {
        pqm::Box box;
        if (pqm::make_box(boxes + (size_t)b * pqm::kBoxFields, box)) live.push_back(box);
    }
    for (int j = 0; j < cols; ++j) {
        pqm::column_init(img, rows, cols, j, obstacle_max, g);
        const double py = pqm::cell_py(m, j);
        for (const pqm::Box &box : live) pqm::stamp_column(g, m, j, py, ms, box);
        pqm::column_sweeps(rows, cols, j, g);
    }
    std::vector<int32_t> rg(cols), h(cols);
    std::vector<int16_t> s(cols), t(cols);
    const int32_t inf = pqm::inf_g(rows, cols);
    for (int i = 0; i < rows; ++i) {
        int32_t *row = g + (size_t)i * cols;
        std::memcpy(rg.data(), row, cols * sizeof(int32_t));
        const int n = pqm::envelope(rg.data(), cols, s.data(), t.data(), h.data());
        for (int q = 0; q < n; ++q) pqm::fill(s.data(), t.data(), h.data(), n, cols, q, rg.data());
        if (d2) std::memcpy(d2 + (size_t)i * cols, rg.data(), cols * sizeof(int32_t));
        float *out = layer + (size_t)i * cols;
        for (int u = 0; u < cols; ++u) out[u] = pqm::layer_value(rg[u], inf * inf, (float)resolution);
    }
    return 0;
}

// the predicate alone: mask[rows * cols] = 1 where a cell centre lies in or on one of the boxes (no base image)
extern "C" int pqm_emu_boxes_mask(int rows, int cols, double resolution, double cx, double cy, const double *boxes,
                                  int k, uint8_t *mask) {
    const pqm::Cells m{rows, cols, resolution, 0.5 * rows * resolution, 0.5 * cols * resolution, cx, cy};
    std::vector<pqm::Box> live;
    for (int b = 0; b < k; ++b) {
        pqm::Box box;
        if (pqm::make_box(boxes + (size_t)b * pqm::kBoxFields, box)) live.push_back(box);
    }
    for (int i = 0; i < rows; ++i)
        for (int j = 0; j < cols; ++j) {
            uint8_t in = 0;
            for (const pqm::Box &box : live)
                in |= pqm::in_box(pqm::cell_px(m, i), pqm::cell_py(m, j), box.x, box.y, box.c, box.s, box.half_l,
                                  box.half_w);
            mask[(size_t)i * cols + j] = in;
        }
    return 0;
}
