// Drives pqp::dropin::ReferenceFrontEndT across a map change, the way a host that gets a new map per tick would:
// a front end constructed on map A gets map B's occupancy image through setOccupancy, and its states and bounds are
// printed next to those of a front end constructed on B's distance layer.
// Input file: rows cols res obstacle_max; <rows*cols floats: layer A>; <rows*cols ints: image B>;
// <rows*cols floats: layer B>; k; 9 rows of k doubles; max_s.
// Output: "refused <0|1>" (setOccupancy of a 1-row image), then for the updated and the fresh front end
// "run <ok> <n>" followed by n lines of s x y heading k f_lb f_ub r_lb r_ub c_lb c_ub.
#include <cstdio>
#include <memory>
#include <vector>

#include "../../include/pqp_reference_path.hpp"
#include "ref_stub.hpp"

typedef pqp::dropin::ReferenceFrontEndT<stub::State, stub::VehicleStateBound> FrontEnd;

static void run(FrontEnd &fe, const pqp::dropin::SplineRows &xs, const pqp::dropin::SplineRows &ys, double max_s) {
    std::vector<stub::State> states;
    std::vector<stub::VehicleStateBound> bounds;
    std::shared_ptr<stub::VehicleStateBound> blocked;
    const bool ok = fe.buildReferenceFromSpline(xs, ys, max_s, 0.15, 0.3, true, &states) &&
                    fe.updateBoundsImproved(xs, ys, &states, &bounds, &blocked);
    std::printf("run %d %zu\n", ok ? 1 : 0, bounds.size());
    for (size_t i = 0; i < bounds.size(); ++i) {
        const stub::State &s = states[i];
        const stub::VehicleStateBound &b = bounds[i];
        std::printf("%.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", s.s, s.x, s.y, s.heading, s.k,
                    b.front.lb, b.front.ub, b.rear.lb, b.rear.ub, b.center.lb, b.center.ub);
    }
}

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    FILE *f = std::fopen(argv[1], "r");
    if (!f) return 2;
    int rows, cols, obstacle_max, k;
    double res, max_s;
    if (std::fscanf(f, "%d %d %lf %d", &rows, &cols, &res, &obstacle_max) != 4) return 2;
    const size_t cells = static_cast<size_t>(rows) * cols;
    std::vector<float> dist_a(cells), dist_b(cells);
    std::vector<unsigned char> img_b(cells);
    for (auto &v : dist_a)
        if (std::fscanf(f, "%f", &v) != 1) return 2;
    for (auto &v : img_b) {
        int p;
        if (std::fscanf(f, "%d", &p) != 1) return 2;
        v = static_cast<unsigned char>(p);
    }
    for (auto &v : dist_b)
        if (std::fscanf(f, "%f", &v) != 1) return 2;
    if (std::fscanf(f, "%d", &k) != 1) return 2;
    pqp::dropin::SplineRows xs, ys;
    std::vector<double> *r[9] = {&xs.x, &xs.a, &xs.b, &xs.c, &xs.y, &ys.a, &ys.b, &ys.c, &ys.y};
    for (auto *row : r) {
        row->resize(k);
        for (auto &v : *row)
            if (std::fscanf(f, "%lf", &v) != 1) return 2;
    }
    ys.x = xs.x;
    if (std::fscanf(f, "%lf", &max_s) != 1) return 2;
    std::fclose(f);
    FrontEnd updated(dist_a.data(), rows, cols, res, 0.0, 0.0);
    const bool refused = !updated.setOccupancy(img_b.data(), 1, cols, res, 0.0, 0.0, obstacle_max);
    std::printf("refused %d\n", refused ? 1 : 0);
    if (!updated.setOccupancy(img_b.data(), rows, cols, res, 0.0, 0.0, obstacle_max)) {
        std::printf("setOccupancy failed: %s\n", updated.lastError().c_str());
        return 1;
    }
    run(updated, xs, ys, max_s);
    FrontEnd fresh(dist_b.data(), rows, cols, res, 0.0, 0.0);
    run(fresh, xs, ys, max_s);
    return 0;
}
