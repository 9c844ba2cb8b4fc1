// Drives pqp::dropin::PathOptimizerT the way the demo drives the reference's PathOptimizer (demo.cpp:196-206): one
// object per plan, constructed with that plan's map, then solve(), getReferencePath(), destruction.
//
//   path_optimizer_test <script>                      one object per `case` line, results on stdout
//   path_optimizer_test <script> bench <warmup> <ticks>  times the first `case` as the demo's tick
//
// Script lines (numbers in text, maps as raw files):
//   params <file>       the raw bytes of a pqp_plan_params (default: the library's defaults)
//   dist <rows> <cols> <resolution> <center_x> <center_y> <file>                 a float32 distance layer
//   occ <rows> <cols> <resolution> <center_x> <center_y> <obstacle_max> <file>   a uint8 occupancy image
//   case <map> <m> <m x> <m y> <start x y heading k> <target x y heading>
// Maps are numbered in the order they appear. Before each solve final_path holds two marker states (x = -7).
// Output per case: "case <i> ok <0|1> status <s> path <rows>", the rows (x y heading k d_k l d_heading s v a), "view
// <k> <length> <states> <bounds> <blocked>", 10 spline rows (x_s.x a b c y, y_s.x a b c y), the states (x y heading k
// s), the bounds and the blocked bound (front, rear, centre: lb ub x y heading each), on a solved plan the path that
// getOptimizedPath makes of the final path's own l, d_heading, k, d_k ("check"), then "error <text>". Last line:
// "pool creates <c> hits <h>".
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/pqp_path_optimizer.hpp"
#include "ref_stub.hpp"

typedef pqp::dropin::PathOptimizerT<stub::State, stub::SlState, stub::VehicleStateBound> Optimizer;

struct MapSpec {
    bool occupancy;
    int rows, cols, obstacle_max;
    double res, cx, cy;
    std::vector<float> dist;
    std::vector<unsigned char> image;
};

struct Case {
    int map;
    std::vector<stub::State> points;
    stub::State start, target;
};

template <class T>
static bool readRaw(const std::string &path, std::vector<T> *v, size_t count) {
    v->resize(count);
    FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) return false;
    const size_t got = std::fread(v->data(), sizeof(T), count, f);
    std::fclose(f);
    return got == count;
}

static Optimizer *construct(const MapSpec &m, const Case &c, const pqp::dropin::PathOptimizerOptions &opt) {
    if (m.occupancy)
        return new Optimizer(c.start, c.target, m.image.data(), m.rows, m.cols, m.res, m.cx, m.cy, m.obstacle_max, opt);
    return new Optimizer(c.start, c.target, m.dist.data(), m.rows, m.cols, m.res, m.cx, m.cy, opt);
}

static void printBound(const stub::VehicleStateBound &b) {
    const stub::VehicleStateBound::SingleBound *s[3] = {&b.front, &b.rear, &b.center};
    for (int i = 0; i < 3; ++i)
        std::printf("%.17g %.17g %.17g %.17g %.17g%s", s[i]->lb, s[i]->ub, s[i]->x, s[i]->y, s[i]->heading,
                    i < 2 ? " " : "\n");
}

static void printRow(const std::vector<double> &r) {
    for (size_t i = 0; i < r.size(); ++i) std::printf("%.17g%s", r[i], i + 1 < r.size() ? " " : "");
    std::printf("\n");
}

static void runCase(int idx, const MapSpec &m, const Case &c, const pqp::dropin::PathOptimizerOptions &opt) {
    Optimizer *po = construct(m, c, opt);
    std::vector<stub::SlState> path(2);
    for (auto &p : path) p.x = p.y = p.heading = p.k = p.d_k = p.l = p.d_heading = -7.0;
    const bool ok = po->solve(c.points, &path);
    std::printf("case %d ok %d status %d path %zu\n", idx, ok ? 1 : 0, po->lastStatus(), path.size());
    for (const auto &p : path)
        std::printf("%.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", p.x, p.y, p.heading, p.k, p.d_k,
                    p.l, p.d_heading, p.s, p.v, p.a);
    const Optimizer::ReferencePathView &v = po->getReferencePath();
    std::printf("view %zu %.17g %zu %zu %d\n", v.x_s.x.size(), v.length, v.reference_states.size(), v.bounds.size(),
                v.blocked ? 1 : 0);
    const pqp::dropin::SplineRows *rows[2] = {&v.x_s, &v.y_s};
    for (const auto *r : rows) {
        printRow(r->x);
        printRow(r->a);
        printRow(r->b);
        printRow(r->c);
        printRow(r->y);
    }
    for (const auto &s : v.reference_states) std::printf("%.17g %.17g %.17g %.17g %.17g\n", s.x, s.y, s.heading, s.k, s.s);
    for (const auto &b : v.bounds) printBound(b);
    if (v.blocked) printBound(*v.blocked);
    if (ok) {  // the construction a failed re-solve uses, applied to the second solution
        const size_t n = path.size();
        std::vector<double> sol(4 * n, 0.0);
        for (size_t i = 0; i < n; ++i) {
            sol[i] = path[i].l;
            sol[n + i] = path[i].d_heading;
            sol[2 * n + i] = path[i].k;
            sol[3 * n + i] = path[i].d_k;
        }
        std::vector<stub::SlState> again;
        pqp::dropin::getOptimizedPath(v.reference_states, sol.data(), n, n, &again);
        std::printf("check %zu\n", again.size());
        for (const auto &p : again)
            std::printf("%.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", p.x, p.y, p.heading, p.k, p.d_k, p.l, p.d_heading);
    }
    std::printf("error %s\n", po->lastError().c_str());
    delete po;
}

static double msSince(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// the demo's tick: construct (a pool hit after the first), solve, getReferencePath, destruct
static void bench(const MapSpec &m, const Case &c, const pqp::dropin::PathOptimizerOptions &opt, int warmup, int ticks) {
    {  // CUDA context and module set-up, so that the first construction times the plan handle alone
        pqp_params sp;
        pqp_default_params(&sp);
        pqp_handle *h = nullptr;
        if (pqp_create(&sp, 31, 1, opt.device, &h) != PQP_OK) {
            std::printf("bench failed: %s\n", pqp_last_error(nullptr));
            return;
        }
        pqp_destroy(h);
    }
    std::vector<double> t;
    double first_construct = 0.0, first_tick = 0.0;
    size_t view_states = 0;
    int status = -1;
    for (int i = 0; i < warmup + ticks + 1; ++i) {
        const auto t0 = std::chrono::steady_clock::now();
        Optimizer *po = construct(m, c, opt);
        if (i == 0) first_construct = msSince(t0);
        std::vector<stub::SlState> path;
        po->solve(c.points, &path);
        view_states = po->getReferencePath().reference_states.size();
        status = po->lastStatus();
        delete po;
        const double ms = msSince(t0);
        if (i == 0) first_tick = ms;
        else if (i > warmup) t.push_back(ms);
    }
    auto &pool = pqp::dropin::PlanHandlePool::instance();
    std::printf("bench status %d states %zu first_construct_ms %.4f first_tick_ms %.4f creates %zu hits %zu\n", status,
                view_states, first_construct, first_tick, pool.creates(), pool.hits());
    std::printf("ticks_ms");
    for (double v : t) std::printf(" %.5f", v);
    std::printf("\n");
}

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    std::ifstream f(argv[1]);
    if (!f) return 2;
    pqp::dropin::PathOptimizerOptions opt;
    std::vector<MapSpec> maps;
    std::vector<Case> cases;
    std::string line;
    while (std::getline(f, line)) {
        std::istringstream in(line);
        std::string kind, file;
        in >> kind;
        if (kind == "params") {
            in >> file;
            std::vector<unsigned char> bytes;
            if (!readRaw(file, &bytes, sizeof(pqp_plan_params))) return 2;
            std::memcpy(&opt.params, bytes.data(), sizeof(pqp_plan_params));
        } else if (kind == "dist" || kind == "occ") {
            MapSpec m;
            m.occupancy = kind == "occ";
            m.obstacle_max = 0;
            in >> m.rows >> m.cols >> m.res >> m.cx >> m.cy;
            if (m.occupancy) in >> m.obstacle_max;
            in >> file;
            const size_t cells = static_cast<size_t>(m.rows) * m.cols;
            if (!in || !(m.occupancy ? readRaw(file, &m.image, cells) : readRaw(file, &m.dist, cells))) return 2;
            maps.push_back(m);
        } else if (kind == "case") {
            Case c;
            size_t n = 0;
            in >> c.map >> n;
            c.points.resize(n);
            for (auto &p : c.points) in >> p.x;
            for (auto &p : c.points) in >> p.y;
            in >> c.start.x >> c.start.y >> c.start.heading >> c.start.k >> c.target.x >> c.target.y >> c.target.heading;
            if (!in || c.map < 0 || c.map >= static_cast<int>(maps.size())) return 2;
            cases.push_back(c);
        }
    }
    if (argc >= 5 && std::string(argv[2]) == "bench") {
        if (cases.empty()) return 2;
        bench(maps[cases[0].map], cases[0], opt, std::atoi(argv[3]), std::atoi(argv[4]));
        return 0;
    }
    for (size_t i = 0; i < cases.size(); ++i) runCase(static_cast<int>(i), maps[cases[i].map], cases[i], opt);
    auto &pool = pqp::dropin::PlanHandlePool::instance();
    std::printf("pool creates %zu hits %zu\n", pool.creates(), pool.hits());
    return 0;
}
