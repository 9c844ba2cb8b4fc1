// pqp_bounds.cu — clearance-bounds kernel and its C ABI (include/pqp_bounds.h).
//
// One thread per (path, reference state, anchor); a warp = one anchor type of 32 consecutive
// states, so its ray-marches walk neighbouring map cells in lock step. The
// float distance layer (2 MB for the demo map) is read through the read-only path and stays in
// the 126 MB L2; per state the kernel reads 32 B of state + its share of the spline and writes
// 48 B of bounds - it is gather-latency bound, not HBM bound (DESIGN.md §5).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>
#include <optional>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/pqp_bounds.h"
#include "pqp_bounds_core.cuh"
#include "pqp_bounds_internal.h"
#include "pqp_collision_core.cuh"
#include "pqp_host_handle.h"
#include "pqp_map_core.cuh"

namespace {

struct BoundsArgs {
    pqb::MapView map;             // the shared map, when map_index is NULL
    const pqb::MapView *table;    // per-path maps: path b reads table[map_index[b]]
    const int32_t *map_index;
    int n_maps;
    pqb::Params prm;
    int batch, n_max, k_max;
    const double *states;
    const int32_t *n;
    const double *spline;
    const int32_t *k;
    double *bounds;
    int32_t *n_valid;
    double *knots;
};

// a path whose map index is out of range gets n_valid = 0 here and is skipped by the clearance kernel
__global__ void init_n_valid_kernel(const int32_t *__restrict__ n, int32_t *__restrict__ n_valid, int batch, int n_max,
                                    const int32_t *__restrict__ map_index, int n_maps) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) {
        int v = n[b];
        if (map_index && !(map_index[b] >= 0 && map_index[b] < n_maps)) v = 0;
        n_valid[b] = v < 0 ? 0 : (v > n_max ? n_max : v);
    }
}

// grid.x covers (path, state) pairs, grid.y the anchor: a warp handles one anchor type of 32
// consecutive states (0.15-0.3 m apart), so its lanes run the same Newton / march phases over
// neighbouring map cells.
__global__ void __launch_bounds__(128) clearance_bounds_kernel(const BoundsArgs a) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)a.batch * a.n_max;
    if (t >= total) return;
    const int anchor = (int)blockIdx.y;
    const int i = (int)(t % a.n_max);
    const int b = (int)(t / a.n_max);
    int nb = a.n[b];
    nb = nb > a.n_max ? a.n_max : nb;
    if (i >= nb) return;
    const double *st = a.states + (size_t)b * PQP_STATE_ROWS * a.n_max;
    const double s = st[i], x = st[a.n_max + i], y = st[2 * a.n_max + i], heading = st[3 * a.n_max + i];
    const double *sb = a.spline + (size_t)b * PQP_SPLINE_ROWS * a.k_max;
    pqb::SplineView sp;
    sp.sx = sb;
    sp.xa = sb + 1 * (size_t)a.k_max; sp.xb = sb + 2 * (size_t)a.k_max; sp.xc = sb + 3 * (size_t)a.k_max; sp.xy = sb + 4 * (size_t)a.k_max;
    sp.ya = sb + 5 * (size_t)a.k_max; sp.yb = sb + 6 * (size_t)a.k_max; sp.yc = sb + 7 * (size_t)a.k_max; sp.yy = sb + 8 * (size_t)a.k_max;
    sp.k = a.k[b] > a.k_max ? a.k_max : a.k[b];
    double lb, ub;
    if (a.map_index) {
        const pqb::MapView *map = pqb::slot_view(a.table, a.n_maps, a.map_index, b);
        if (!map) return;
        pqb::anchor_bounds(*map, a.prm, sp, s, x, y, heading, anchor, lb, ub);
    } else {
        pqb::anchor_bounds(a.map, a.prm, sp, s, x, y, heading, anchor, lb, ub);
    }
    double *ob = a.bounds + (size_t)b * PQP_BOUND_ROWS * a.n_max;
    ob[(size_t)(2 * anchor) * a.n_max + i] = lb;
    ob[(size_t)(2 * anchor + 1) * a.n_max + i] = ub;
    if (anchor < 2) {
        if (a.knots) {
            double *kb = a.knots + (size_t)b * PQP_NFIELDS * a.n_max;
            const int f = anchor == 0 ? PQP_F_B0_LB : PQP_F_B1_LB;
            kb[(size_t)f * a.n_max + i] = lb;
            kb[(size_t)(f + 1) * a.n_max + i] = ub;
        }
        // isEqual(bound[0], bound[1]) -> "Path is blocked" (reference_path_impl.cpp:216-220)
        if (fabs(ub - lb) < a.prm.epsilon) atomicMin(a.n_valid + b, i);
    }
}

struct StatesArgs {
    int batch, n_max, k_max;
    const double *spline;
    const int32_t *k;
    const double *max_s;
    double ds_small, ds_large;
    int dynamic;
    double *states, *curvature, *knots;
    int32_t *n, *total;
};

// one thread per path: the walk is sequential in s (each step depends on the curvature at the last)
__global__ void __launch_bounds__(64) reference_states_kernel(const StatesArgs a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.batch) return;
    const double *sb = a.spline + (size_t)b * PQP_SPLINE_ROWS * a.k_max;
    pqb::SplineView sp;
    sp.sx = sb;
    sp.xa = sb + 1 * (size_t)a.k_max; sp.xb = sb + 2 * (size_t)a.k_max; sp.xc = sb + 3 * (size_t)a.k_max; sp.xy = sb + 4 * (size_t)a.k_max;
    sp.ya = sb + 5 * (size_t)a.k_max; sp.yb = sb + 6 * (size_t)a.k_max; sp.yc = sb + 7 * (size_t)a.k_max; sp.yy = sb + 8 * (size_t)a.k_max;
    sp.k = a.k[b] > a.k_max ? a.k_max : a.k[b];
    double *st = a.states + (size_t)b * PQP_STATE_ROWS * a.n_max;
    double *cv = a.curvature + (size_t)b * a.n_max;
    const int total = pqb::build_states(sp, a.max_s[b], a.ds_small, a.ds_large, a.dynamic != 0, a.n_max, a.total != nullptr, st, cv);
    const int nb = total < a.n_max ? total : a.n_max;
    a.n[b] = nb;
    if (a.total) a.total[b] = total;
    if (a.knots) {
        double *kb = a.knots + (size_t)b * PQP_NFIELDS * a.n_max;
        for (int i = 0; i < nb; ++i) {
            kb[(size_t)PQP_F_S * a.n_max + i] = st[i];
            kb[(size_t)PQP_F_KREF * a.n_max + i] = cv[i];
            kb[(size_t)PQP_F_L * a.n_max + i] = 0.0;
            kb[(size_t)PQP_F_PSI * a.n_max + i] = 0.0;
            kb[(size_t)PQP_F_K * a.n_max + i] = cv[i];
        }
    }
}

struct CollisionArgs {
    pqb::MapView map;             // the shared map, when map_index is NULL
    const pqb::MapView *table;    // per-path maps: path b reads table[map_index[b]]
    const int32_t *map_index;
    int n_maps;
    pqc::Footprint fp;
    int n_max, row_stride;
    const double *poses;
    const int32_t *n;
    int32_t *first_hit;
    uint8_t *state_free;
    double *clearance;
};

constexpr int kCollisionThreads = 128;

// one CTA per path: the threads stride over its states and a block min-reduction gives the first state that is
// not free (no atomics, so no initialisation launch, and the result does not depend on thread timing)
__global__ void __launch_bounds__(kCollisionThreads) collision_check_kernel(const CollisionArgs a) {
    __shared__ int warp_min[kCollisionThreads / 32];
    const int b = blockIdx.x;
    int nb = a.n[b];
    nb = nb < 0 ? 0 : (nb > a.n_max ? a.n_max : nb);
    pqb::MapView m = a.map;
    if (a.map_index) {
        const pqb::MapView *slot = pqb::slot_view(a.table, a.n_maps, a.map_index, b);
        if (slot) m = *slot;
        else nb = -1;  // reads no map; every state gets the i >= n outputs
    }
    const double *x = a.poses + (size_t)b * a.row_stride * a.n_max, *y = x + a.n_max, *h = y + a.n_max;
    int hit = nb < 0 ? -1 : nb;
    for (int i = threadIdx.x; i < a.n_max; i += kCollisionThreads) {
        bool free_ = false;
        double c = 0.0;
        if (i < nb) {
            free_ = pqc::state_free(m, a.fp, x[i], y[i], h[i], c);
            if (!free_ && i < hit) hit = i;
        }
        if (a.state_free) a.state_free[(size_t)b * a.n_max + i] = free_ ? 1 : 0;
        if (a.clearance) a.clearance[(size_t)b * a.n_max + i] = c;
    }
    hit = __reduce_min_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0) warp_min[threadIdx.x >> 5] = hit;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kCollisionThreads / 32; ++w) hit = warp_min[w] < hit ? warp_min[w] : hit;
        a.first_hit[b] = hit;
    }
}

}  // namespace

// The exact Euclidean distance transform of pqp_bounds_set_occupancy* (pqp_map_core.cuh), in place in the
// distance layer: the column pass writes int32 g over the layer, the row pass reads its row of g into shared
// memory and writes the row's floats back. Named namespace: the kernels keep stable names in profiles.
namespace pqm {

constexpr int kEdtColumnThreads = 128;
constexpr int kEdtRowThreads = 64;

// Table entries first .. first + n - 1 of a slot update: `meta` with slot first + i's layer and centre i. Passed by
// value, so the entries a launch writes are fixed when it is enqueued (PQP_MAP_TABLE_CHUNK * 16 B of parameters).
struct TableWrite {
    pqb::MapView *table;
    pqb::MapView meta;  // dist: the layer of slot `first`
    size_t slot_cells;
    int first, n;
    double cx[PQP_MAP_TABLE_CHUNK], cy[PQP_MAP_TABLE_CHUNK];
};

__global__ void map_table_kernel(const TableWrite w) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w.n) return;
    pqb::MapView m = w.meta;
    m.dist += (size_t)i * w.slot_cells;
    m.cx = w.cx[i];
    m.cy = w.cy[i];
    w.table[w.first + i] = m;
}

// The column pass's stamping argument: NoBoxes for the plain images, SlotBoxes for pqp_bounds_set_occupancy_boxes*.
struct NoBoxes {};
struct SlotBoxes {
    const pqb::MapView *table;  // the slots' table entries from the first slot on (their centres), written before
    const double *boxes;        // [count][k_max][kBoxFields]
    const int32_t *k;           // [count], clamped to [0, k_max]; not read when k_max = 0
    int k_max;
    size_t img_stride;          // bytes from one slot's base image to the next: 0 when every slot shares one
};

// The box instantiation's work for column j of slot blockIdx.y: base image into g, the slot's boxes stamped in chunks
// of one box per thread, then the two sweeps. Each chunk is loaded once per block (one sincos per box) and only the
// boxes that can reach the block's columns are kept.
__device__ __forceinline__ void stamped_column(const uint8_t *__restrict__ img, int rows, int cols, int obstacle_max,
                                               int32_t *__restrict__ g, size_t slot_cells, const SlotBoxes &sb) {
    __shared__ pqm::Box live[kEdtColumnThreads];
    __shared__ int n_live;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const size_t y = blockIdx.y;
    img += y * sb.img_stride;
    g += y * slot_cells;
    int kb = sb.k_max > 0 ? sb.k[y] : 0;
    kb = kb < 0 ? 0 : (kb > sb.k_max ? sb.k_max : kb);
    if (kb == 0) {  // uniform in the block: the plain column pass
        if (j < cols) pqm::column_pass(img, rows, cols, j, obstacle_max, g);
        return;
    }
    const pqb::MapView mv = sb.table[y];
    const pqm::Cells m{rows, cols, mv.res, mv.half_lx, mv.half_ly, mv.cx, mv.cy};
    const double ms = pqm::map_slack(m);
    const int j0 = blockIdx.x * blockDim.x, j1 = (j0 + (int)blockDim.x < cols ? j0 + (int)blockDim.x : cols) - 1;
    const double py_hi = pqm::cell_py(m, j0) + ms, py_lo = pqm::cell_py(m, j1) - ms;
    const double py = pqm::cell_py(m, j < cols ? j : j1);
    if (j < cols) pqm::column_init(img, rows, cols, j, obstacle_max, g);
    const double *bs = sb.boxes + y * (size_t)sb.k_max * pqm::kBoxFields;
    for (int first = 0; first < kb; first += kEdtColumnThreads) {
        if (threadIdx.x == 0) n_live = 0;
        __syncthreads();
        const int b = first + threadIdx.x;
        pqm::Box box;
        if (b < kb && pqm::make_box(bs + (size_t)b * pqm::kBoxFields, box) && pqm::box_reaches(box, py_lo, py_hi))
            live[atomicAdd(&n_live, 1)] = box;  // the order does not matter: stamps only ever set g = 0
        __syncthreads();
        if (j < cols)
            for (int q = 0; q < n_live; ++q) pqm::stamp_column(g, m, j, py, ms, live[q]);
        __syncthreads();
    }
    if (j < cols) pqm::column_sweeps(rows, cols, j, g);
}

// one thread per column of image blockIdx.y: consecutive threads read consecutive bytes of a row. Images are
// rows * cols bytes apart, their g slot_cells int32 apart (in the layers of consecutive slots). A one-image update
// also writes its slot's table entry (`entry_dst`, NULL for none) here, so it costs no launch of its own. The SlotBoxes
// instantiation stamps each slot's boxes into its image first (stamped_column; entry_dst is NULL there).
template <class Stamp>
__global__ void __launch_bounds__(kEdtColumnThreads) edt_column_kernel(const uint8_t *__restrict__ img, int rows, int cols,
                                                                        int obstacle_max, int32_t *__restrict__ g,
                                                                        size_t slot_cells, pqb::MapView *entry_dst,
                                                                        const pqb::MapView entry, const Stamp stamp) {
    if constexpr (std::is_same<Stamp, SlotBoxes>::value) {
        stamped_column(img, rows, cols, obstacle_max, g, slot_cells, stamp);
    } else {
        const int j = blockIdx.x * blockDim.x + threadIdx.x;
        const size_t y = blockIdx.y;
        if (entry_dst && j == 0 && y == 0) *entry_dst = entry;
        if (j < cols) pqm::column_pass(img + y * rows * cols, rows, cols, j, obstacle_max, g + y * slot_cells);
    }
}

// one block per row of image blockIdx.y: the block loads the row's g, thread 0 builds the lower envelope, the block
// fills d2 per envelope parabola and converts it to the layer's floats
__global__ void __launch_bounds__(kEdtRowThreads) edt_row_kernel(void *layers, size_t slot_cells, int rows, int cols,
                                                                 float res) {
    extern __shared__ int4 edt_smem[];
    int32_t *g = reinterpret_cast<int32_t *>(edt_smem);
    int32_t *h = g + cols;
    int16_t *s = reinterpret_cast<int16_t *>(h + cols);
    int16_t *t = s + cols;
    __shared__ int n_env;
    void *layer = static_cast<int32_t *>(layers) + blockIdx.y * slot_cells;
    const size_t row = (size_t)blockIdx.x * cols;
    const int32_t *gin = static_cast<const int32_t *>(layer) + row;
    for (int u = threadIdx.x; u < cols; u += blockDim.x) g[u] = gin[u];
    __syncthreads();
    if (threadIdx.x == 0) n_env = pqm::envelope(g, cols, s, t, h);
    __syncthreads();
    const int n = n_env;
    for (int k = threadIdx.x; k < n; k += blockDim.x) pqm::fill(s, t, h, n, cols, k, g);
    __syncthreads();
    const int32_t inf = pqm::inf_g(rows, cols);
    float *out = static_cast<float *>(layer) + row;
    for (int u = threadIdx.x; u < cols; u += blockDim.x) out[u] = pqm::layer_value(g[u], inf * inf, res);
}

}  // namespace pqm

struct pqp_bounds_handle {
    int device = 0;
    int n_maps = 1;
    std::vector<pqb::MapView> maps;  // the slots' metadata as the host calls left them (slot 0: the unmapped calls' map)
    pqb::Params prm{};
    float *d_dist = nullptr;          // [n_maps][cap_cells] distance layers
    size_t cap_cells = 0;             // cells per slot: the largest map the handle was created with
    uint8_t *d_occ = nullptr;         // [n_maps][cap_cells] staging of the host set_occupancy calls' images
    double *d_boxes = nullptr;        // [PQP_MAX_BOXES][PQP_BOX_FIELDS] staging of the host set_occupancy_boxes call
    int32_t *d_box_k = nullptr;       // [n_maps] its box counts
    pqb::MapView *d_table = nullptr;  // [n_maps] the slots' metadata as the mapped kernels read it, in stream order
    std::unique_ptr<pqm::TableWrite> tw{new (std::nothrow) pqm::TableWrite};  // parameters of map_table_kernel
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // staging for the host-pointer call (grown on demand)
    double *d_states = nullptr, *d_spline = nullptr, *d_bounds = nullptr, *d_knots = nullptr;
    int32_t *d_n = nullptr, *d_k = nullptr, *d_nvalid = nullptr, *d_map_index = nullptr;
    double *d_maxs = nullptr, *d_curv = nullptr;
    int32_t *d_total = nullptr;
    int32_t *d_hit = nullptr;   // the host collision check's outputs (its poses and n go to d_states, d_n)
    uint8_t *d_free = nullptr;
    double *d_clear = nullptr;
    pqc::Footprint footprint{};  // of prm, at create
    bool timed = false;
    std::string err;
    pqp::Resources res;  // last member: releasing clears the members above
};

namespace pqb {
const MapView *handle_map(const pqp_bounds_handle *h) { return h ? &h->maps[0] : nullptr; }
int handle_device(const pqp_bounds_handle *h) { return h ? h->device : -1; }
const MapView *handle_table(const pqp_bounds_handle *h) { return h ? h->d_table : nullptr; }
int handle_map_count(const pqp_bounds_handle *h) { return h ? h->n_maps : 0; }
}  // namespace pqb

namespace {

thread_local std::string g_bounds_create_error;

using pqp::fail;

int validate(pqp_bounds_handle *h, const pqp_bounds_in *in, const pqp_bounds_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || in->batch <= 0 || in->n_max <= 0 || in->k_max < 3 || !in->states || !in->n || !in->spline ||
        !in->k || !out->bounds || !out->n_valid)
        return fail(h->err, PQP_E_INVALID, "pqp_bounds: null pointer or non-positive size (batch, n_max > 0, k_max >= 3)");
    return PQP_OK;
}

// map_index: NULL for the shared map (slot 0 as the host last set it), else [batch] slot per path on the device
int launch(pqp_bounds_handle *h, const pqp_bounds_in *in, const int32_t *map_index, const pqp_bounds_out *out,
           cudaStream_t s) {
    BoundsArgs a;
    a.map = h->maps[0];
    a.table = h->d_table;
    a.map_index = map_index;
    a.n_maps = h->n_maps;
    a.prm = h->prm;
    a.batch = in->batch;
    a.n_max = in->n_max;
    a.k_max = in->k_max;
    a.states = in->states;
    a.n = in->n;
    a.spline = in->spline;
    a.k = in->k;
    a.bounds = out->bounds;
    a.n_valid = out->n_valid;
    a.knots = out->knots;
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, s));
    init_n_valid_kernel<<<(in->batch + 255) / 256, 256, 0, s>>>(in->n, out->n_valid, in->batch, in->n_max, map_index,
                                                                 h->n_maps);
    const long long total = (long long)in->batch * in->n_max;
    const long long blocks = (total + 127) / 128;
    if (blocks > 0x7fffffffLL) return fail(h->err, PQP_E_INVALID, "pqp_bounds: batch * n_max too large for one launch");
    clearance_bounds_kernel<<<dim3((unsigned)blocks, 3), 128, 0, s>>>(a);
    PQP_CUDA(h->err, cudaGetLastError());
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, s));
    h->timed = true;
    return PQP_OK;
}

pqb::MapView make_view(const float *dist, int rows, int cols, double res, double cx, double cy) {
    pqb::MapView m;
    m.dist = dist;
    m.rows = rows;
    m.cols = cols;
    m.res = res;
    m.inv_res = 1.0 / res;
    m.half_lx = 0.5 * rows * res;
    m.half_ly = 0.5 * cols * res;
    m.cx = cx;
    m.cy = cy;
    return m;
}

float *slot_layer(pqp_bounds_handle *h, int slot) { return h->d_dist + (size_t)slot * h->cap_cells; }

// table entries first .. first + count - 1: `meta` (dist: slot first's layer) with centre i = (cx[i], cy[i]), in
// launches of PQP_MAP_TABLE_CHUNK entries
int write_table(pqp_bounds_handle *h, int first, int count, const pqb::MapView &meta, const double *cx, const double *cy,
                cudaStream_t s) {
    pqm::TableWrite &w = *h->tw;
    for (int done = 0; done < count; done += PQP_MAP_TABLE_CHUNK) {
        const int n = count - done < PQP_MAP_TABLE_CHUNK ? count - done : PQP_MAP_TABLE_CHUNK;
        w.table = h->d_table;
        w.meta = meta;
        w.meta.dist = meta.dist + (size_t)done * h->cap_cells;
        w.slot_cells = h->cap_cells;
        w.first = first + done;
        w.n = n;
        for (int i = 0; i < n; ++i) {
            w.cx[i] = cx[done + i];
            w.cy[i] = cy[done + i];
        }
        pqm::map_table_kernel<<<(n + 127) / 128, 128, 0, s>>>(w);
        PQP_CUDA(h->err, cudaGetLastError());
    }
    return PQP_OK;
}

// what pqp_bounds_set_map* and pqp_bounds_set_occupancy* accept; a refused map leaves the handle's maps untouched
int validate_map(pqp_bounds_handle *h, const void *m, int rows, int cols, double res, double cx, double cy,
                 const void *data, const char *what) {
    if (!h) return PQP_E_INVALID;
    std::string why;
    if (!m || !data) why = "null map or layer";
    else if (rows < 2 || cols < 2) why = "rows, cols >= 2 required";
    else if ((size_t)rows * (size_t)cols > h->cap_cells) why = "rows * cols exceeds the cells the handle was created with";
    else if (!(res > 0.0) || !std::isfinite(res)) why = "resolution must be finite and > 0";
    else if (!std::isfinite(cx) || !std::isfinite(cy)) why = "centre must be finite";
    return why.empty() ? PQP_OK : fail(h->err, PQP_E_INVALID, std::string(what) + ": " + why);
}

int validate_slots(pqp_bounds_handle *h, long long first, long long count, const char *what) {
    if (first < 0 || count < 1 || first + count > h->n_maps)
        return fail(h->err, PQP_E_INVALID, std::string(what) + ": slots " + std::to_string(first) + " .. " +
                                               std::to_string(first + count - 1) + " outside [0, " +
                                               std::to_string(h->n_maps) + ")");
    return PQP_OK;
}

// One pqp_bounds_set_occupancy* call: the images of `stack` into slots first .. first + count - 1. `boxed`: the box
// call, which stamps each slot's `boxes` into the base image(s) (one shared when shared_base is 1) and refuses a NULL
// `boxes`. `single`: the one-image call, a count-1 stack at slot 0, whose column pass writes the slot's table entry.
struct Occupancy {
    int first;
    const pqp_occupancy_stack *stack;
    bool boxed;
    int shared_base;
    const pqp_obstacle_boxes *boxes;
    bool single;
};

// what every pqp_bounds_set_occupancy* call refuses, in this order; `host`: the host form, which can read k
int validate(pqp_bounds_handle *h, const Occupancy &r, bool host, const char *what) {
    if (!h) return PQP_E_INVALID;
    const pqp_occupancy_stack *st = r.stack;
    if (!st || !st->cells || !st->center_x || !st->center_y)
        return fail(h->err, PQP_E_INVALID,
                    std::string(what) + (r.single ? ": null map or layer" : ": null stack, image or centres"));
    int rc = validate_slots(h, r.first, st->count, what);
    for (int i = 0; rc == PQP_OK && i < st->count; ++i)
        rc = validate_map(h, st, st->rows, st->cols, st->resolution, st->center_x[i], st->center_y[i], st->cells, what);
    if (rc != PQP_OK) return rc;
    if (st->rows > pqm::kMaxSide || st->cols > pqm::kMaxSide)
        return fail(h->err, PQP_E_INVALID, std::string(what) + ": rows and cols must be <= 16384 for the distance transform");
    if (!r.boxed) return PQP_OK;
    std::string why;
    const pqp_obstacle_boxes *boxes = r.boxes;
    if (r.shared_base != 0 && r.shared_base != 1) why = "shared_base must be 0 or 1";
    else if (!boxes) why = "null boxes";
    else if (boxes->k_max < 0) why = "k_max must be >= 0";
    else if ((long long)st->count * boxes->k_max > PQP_MAX_BOXES)
        why = "count * k_max = " + std::to_string((long long)st->count * boxes->k_max) + " exceeds PQP_MAX_BOXES (" +
              std::to_string(PQP_MAX_BOXES) + ")";
    else if (boxes->k_max > 0 && (!boxes->k || !boxes->boxes)) why = "null k or boxes with k_max > 0";
    else if (host && boxes->k_max > 0)
        for (int i = 0; i < st->count && why.empty(); ++i)
            if (boxes->k[i] < 0 || boxes->k[i] > boxes->k_max)
                why = "k[" + std::to_string(i) + "] = " + std::to_string(boxes->k[i]) + " outside [0, k_max]";
    return why.empty() ? PQP_OK : fail(h->err, PQP_E_INVALID, std::string(what) + ": " + why);
}

// every pqp_bounds_set_occupancy* entry point; `stream` empty for the host forms, which stage the image(s), k and the
// boxes into the handle's buffers, run on the handle's stream and wait
int occupancy(pqp_bounds_handle *h, const Occupancy &r, std::optional<cudaStream_t> stream, const char *what) {
    int rc = validate(h, r, !stream, what);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    const pqp_occupancy_stack &st = *r.stack;
    const cudaStream_t s = stream ? *stream : h->stream;
    const int k_max = r.boxed ? r.boxes->k_max : 0;
    const uint8_t *cells = st.cells;
    const int32_t *k = r.boxed ? r.boxes->k : nullptr;
    const double *xs = r.boxed ? r.boxes->boxes : nullptr;
    if (!stream) {
        // the images are consecutive in the slots' staging: count * rows * cols <= count * cap_cells bytes
        uint8_t *staging = h->d_occ + (size_t)r.first * h->cap_cells;
        const size_t bytes = (size_t)(r.shared_base ? 1 : st.count) * st.rows * st.cols;
        const size_t n_box = (size_t)st.count * k_max;
        PQP_CUDA(h->err, cudaMemcpyAsync(staging, st.cells, bytes, cudaMemcpyHostToDevice, s));
        if (n_box) {
            PQP_CUDA(h->err, cudaMemcpyAsync(h->d_box_k, k, st.count * sizeof(int32_t), cudaMemcpyHostToDevice, s));
            PQP_CUDA(h->err, cudaMemcpyAsync(h->d_boxes, xs, n_box * PQP_BOX_FIELDS * sizeof(double),
                                             cudaMemcpyHostToDevice, s));
        }
        cells = staging;
        k = h->d_box_k;
        xs = h->d_boxes;
    }
    float *layer = slot_layer(h, r.first);
    const pqb::MapView meta = make_view(layer, st.rows, st.cols, st.resolution, r.single ? st.center_x[0] : 0.0,
                                        r.single ? st.center_y[0] : 0.0);
    // the box instantiation of the column pass reads the slots' centres from their table entries: those go first
    if (!r.single) {
        rc = write_table(h, r.first, st.count, meta, st.center_x, st.center_y, s);
        if (rc != PQP_OK) return rc;
    }
    const size_t smem = (size_t)pqm::kRowSmemPerCol * st.cols;
    // the dynamic share plus the kernel's static n_env may pass the 48 KB default at any width: always opt in
    PQP_CUDA(h->err, cudaFuncSetAttribute(pqm::edt_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((st.cols + pqm::kEdtColumnThreads - 1) / pqm::kEdtColumnThreads, st.count);
    int32_t *g = reinterpret_cast<int32_t *>(layer);
    if (r.boxed)
        pqm::edt_column_kernel<<<grid, pqm::kEdtColumnThreads, 0, s>>>(
            cells, st.rows, st.cols, st.obstacle_max, g, h->cap_cells, nullptr, meta,
            pqm::SlotBoxes{h->d_table + r.first, xs, k, k_max, r.shared_base ? 0 : (size_t)st.rows * st.cols});
    else
        pqm::edt_column_kernel<<<grid, pqm::kEdtColumnThreads, 0, s>>>(cells, st.rows, st.cols, st.obstacle_max, g,
                                                                       h->cap_cells, r.single ? h->d_table : nullptr,
                                                                       meta, pqm::NoBoxes{});
    PQP_CUDA(h->err, cudaGetLastError());
    pqm::edt_row_kernel<<<dim3(st.rows, st.count), pqm::kEdtRowThreads, smem, s>>>(layer, h->cap_cells, st.rows, st.cols,
                                                                                   (float)st.resolution);
    PQP_CUDA(h->err, cudaGetLastError());
    for (int i = 0; i < st.count; ++i)
        h->maps[r.first + i] = make_view(slot_layer(h, r.first + i), st.rows, st.cols, st.resolution, st.center_x[i],
                                         st.center_y[i]);
    if (!stream) PQP_CUDA(h->err, cudaStreamSynchronize(s));
    return PQP_OK;
}

// pqp_bounds_set_occupancy(_device): `occ` as a count-1 stack at slot 0 with its centre
int occupancy_image(pqp_bounds_handle *h, const pqp_occupancy_map *occ, std::optional<cudaStream_t> stream,
                    const char *what) {
    pqp_occupancy_stack st{};
    if (occ) st = {1, occ->rows, occ->cols, occ->resolution, &occ->center_x, &occ->center_y, occ->cells, occ->obstacle_max};
    return occupancy(h, {0, occ ? &st : nullptr, false, 0, nullptr, true}, stream, what);
}

int create(const pqp_bounds_map *maps, int n_maps, const pqp_bounds_params *params, int32_t device,
           pqp_bounds_handle **out, const char *what) {
    if (!out) return PQP_E_INVALID;
    *out = nullptr;
    if (n_maps < 1 || n_maps > PQP_MAX_MAP_SLOTS)
        return fail(g_bounds_create_error, PQP_E_INVALID, std::string(what) + ": 1 <= n_maps <= 65535 required");
    size_t cap = 0;
    for (int i = 0; i < n_maps; ++i) {
        if (!maps || !maps[i].distance || maps[i].rows < 2 || maps[i].cols < 2 || !(maps[i].resolution > 0.0))
            return fail(g_bounds_create_error, PQP_E_INVALID,
                        std::string(what) + ": map needs rows, cols >= 2, resolution > 0 and a distance layer");
        const size_t cells = (size_t)maps[i].rows * maps[i].cols;
        cap = cells > cap ? cells : cap;
    }
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count)
        return fail(g_bounds_create_error, PQP_E_NO_DEVICE, std::string(what) + ": no CUDA device (there is no CPU fallback)");
    pqp_bounds_handle *h = new (std::nothrow) pqp_bounds_handle();
    if (!h || !h->tw) {
        delete h;
        return fail(g_bounds_create_error, PQP_E_CUDA, std::string(what) + ": out of host memory");
    }
    h->device = h->res.device = device;
    pqp_bounds_params dflt;
    pqp_bounds_default_params(&dflt);
    const pqp_bounds_params &p = params ? *params : dflt;
    h->prm.front_length = p.front_length;
    h->prm.rear_length = p.rear_length;
    h->prm.car_width = p.car_width;
    h->prm.safety_margin = p.safety_margin;
    h->prm.epsilon = p.epsilon;
    // CollisionChecker's constructor (collision_checker.cpp:9-15)
    h->footprint = pqc::car_footprint(p.car_width, fabs(p.rear_length), p.front_length);
    h->n_maps = n_maps;
    h->cap_cells = cap;
    pqp::DeviceGuard guard_(device);
    const int rc = [&]() -> int {
        std::string &err = g_bounds_create_error;
        const size_t total = (size_t)n_maps * cap;
        const cudaError_t e = h->res.alloc(h->d_dist, total);
        if (e != cudaSuccess)
            return fail(err, PQP_E_CUDA, std::string(what) + ": cannot allocate " + std::to_string(n_maps) + " slots of " +
                                             std::to_string(cap) + " cells (" + std::to_string(total * sizeof(float)) +
                                             " bytes of layers): " + cudaGetErrorString(e));
        PQP_CUDA(err, h->res.alloc(h->d_occ, total));
        PQP_CUDA(err, h->res.alloc(h->d_boxes, (size_t)PQP_MAX_BOXES * PQP_BOX_FIELDS));
        PQP_CUDA(err, h->res.alloc(h->d_box_k, (size_t)n_maps));
        PQP_CUDA(err, h->res.alloc(h->d_table, (size_t)n_maps));
        h->maps.resize(n_maps);
        for (int i = 0; i < n_maps; ++i) {
            const pqp_bounds_map &m = maps[i];
            h->maps[i] = make_view(slot_layer(h, i), m.rows, m.cols, m.resolution, m.center_x, m.center_y);
            PQP_CUDA(err, cudaMemcpy(slot_layer(h, i), m.distance, (size_t)m.rows * m.cols * sizeof(float),
                                     cudaMemcpyHostToDevice));
        }
        PQP_CUDA(err, cudaMemcpy(h->d_table, h->maps.data(), n_maps * sizeof(pqb::MapView), cudaMemcpyHostToDevice));
        PQP_CUDA(err, h->res.stream(h->stream));
        PQP_CUDA(err, h->res.event(h->ev0));
        PQP_CUDA(err, h->res.event(h->ev1));
        return PQP_OK;
    }();
    if (rc != PQP_OK) {
        pqp_bounds_destroy(h);
        return rc;
    }
    *out = h;
    return PQP_OK;
}

// pqp_bounds_set_map(_slot)(_device); `stream` empty: the host forms, which run on the handle's stream and wait
int set_map_slot(pqp_bounds_handle *h, int slot, const pqp_bounds_map *map, std::optional<cudaStream_t> stream,
                 const char *what) {
    if (!h) return PQP_E_INVALID;
    int rc = validate_slots(h, slot, 1, what);
    if (rc != PQP_OK) return rc;
    rc = map ? validate_map(h, map, map->rows, map->cols, map->resolution, map->center_x, map->center_y, map->distance,
                            what)
             : validate_map(h, nullptr, 0, 0, 0.0, 0.0, 0.0, nullptr, what);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    const cudaStream_t s = stream ? *stream : h->stream;
    const size_t cells = (size_t)map->rows * map->cols;
    PQP_CUDA(h->err, cudaMemcpyAsync(slot_layer(h, slot), map->distance, cells * sizeof(float), cudaMemcpyDefault, s));
    const pqb::MapView m = make_view(slot_layer(h, slot), map->rows, map->cols, map->resolution, map->center_x,
                                     map->center_y);
    rc = write_table(h, slot, 1, m, &map->center_x, &map->center_y, s);
    if (rc != PQP_OK) return rc;
    h->maps[slot] = m;
    if (!stream) PQP_CUDA(h->err, cudaStreamSynchronize(s));
    return PQP_OK;
}

int get_map_slot(pqp_bounds_handle *h, int slot, pqp_bounds_map *meta, float *distance, const char *what) {
    if (!h) return PQP_E_INVALID;
    if (!meta) return fail(h->err, PQP_E_INVALID, std::string(what) + ": null metadata");
    const int rc = validate_slots(h, slot, 1, what);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    const pqb::MapView &m = h->maps[slot];
    meta->rows = m.rows;
    meta->cols = m.cols;
    meta->resolution = m.res;
    meta->center_x = m.cx;
    meta->center_y = m.cy;
    meta->distance = nullptr;
    if (distance) {
        PQP_CUDA(h->err, cudaDeviceSynchronize());
        PQP_CUDA(h->err, cudaMemcpy(distance, m.dist, (size_t)m.rows * m.cols * sizeof(float), cudaMemcpyDeviceToHost));
    }
    return PQP_OK;
}

// every pqp_bounds_compute* entry point: `mapped` for the mapped forms (path b on slot map_index[b]), `stream` empty
// for the host forms, which stage the inputs into the handle's buffers, run on the handle's stream, copy the outputs
// back and wait
int compute(pqp_bounds_handle *h, const pqp_bounds_in *in, bool mapped, const int32_t *map_index,
            const pqp_bounds_out *out, std::optional<cudaStream_t> stream) {
    int rc = validate(h, in, out);
    if (rc != PQP_OK) return rc;
    if (mapped && !map_index)
        return fail(h->err, PQP_E_INVALID,
                    stream ? "pqp_bounds_compute_mapped_device: null map_index" : "pqp_bounds_compute_mapped: null map_index");
    pqp::DeviceGuard guard_(h->device);
    if (stream) return launch(h, in, map_index, out, *stream);
    const size_t B = in->batch, ns = B * PQP_STATE_ROWS * in->n_max, nsp = B * PQP_SPLINE_ROWS * in->k_max;
    const size_t nb = B * PQP_BOUND_ROWS * in->n_max, nk = out->knots ? B * PQP_NFIELDS * in->n_max : 0;
    PQP_CUDA(h->err, h->res.grow(h->d_states, ns));
    PQP_CUDA(h->err, h->res.grow(h->d_bounds, nb));
    PQP_CUDA(h->err, h->res.grow(h->d_spline, nsp));
    if (nk) PQP_CUDA(h->err, h->res.grow(h->d_knots, nk));
    PQP_CUDA(h->err, h->res.grow(h->d_n, B));
    PQP_CUDA(h->err, h->res.grow(h->d_k, B));
    PQP_CUDA(h->err, h->res.grow(h->d_nvalid, B));
    if (mapped) PQP_CUDA(h->err, h->res.grow(h->d_map_index, B));
    cudaStream_t s = h->stream;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_states, in->states, ns * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_spline, in->spline, nsp * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_n, in->n, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_k, in->k, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    if (nk) PQP_CUDA(h->err, cudaMemcpyAsync(h->d_knots, out->knots, nk * sizeof(double), cudaMemcpyHostToDevice, s));
    if (mapped)
        PQP_CUDA(h->err, cudaMemcpyAsync(h->d_map_index, map_index, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    pqp_bounds_in din = *in;
    din.states = h->d_states;
    din.spline = h->d_spline;
    din.n = h->d_n;
    din.k = h->d_k;
    pqp_bounds_out dout;
    dout.bounds = h->d_bounds;
    dout.n_valid = h->d_nvalid;
    dout.knots = nk ? h->d_knots : nullptr;
    rc = launch(h, &din, mapped ? h->d_map_index : nullptr, &dout, s);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(h->err, cudaMemcpyAsync(out->bounds, h->d_bounds, nb * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->n_valid, h->d_nvalid, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (nk) PQP_CUDA(h->err, cudaMemcpyAsync(out->knots, h->d_knots, nk * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaStreamSynchronize(s));
    return PQP_OK;
}

int launch_collision(pqp_bounds_handle *h, const pqp_collision_in *in, const int32_t *map_index,
                     const pqp_collision_out *out, cudaStream_t s) {
    CollisionArgs a;
    a.map = h->maps[0];
    a.table = h->d_table;
    a.map_index = map_index;
    a.n_maps = h->n_maps;
    a.fp = h->footprint;
    a.n_max = in->n_max;
    a.row_stride = in->row_stride;
    a.poses = in->poses;
    a.n = in->n;
    a.first_hit = out->first_hit;
    a.state_free = out->state_free;
    a.clearance = out->clearance;
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, s));
    collision_check_kernel<<<in->batch, kCollisionThreads, 0, s>>>(a);
    PQP_CUDA(h->err, cudaGetLastError());
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, s));
    h->timed = true;
    return PQP_OK;
}

// every pqp_bounds_collision_check* entry point, as compute: `mapped` for the mapped forms, `stream` empty for the
// host forms
int collision_check(pqp_bounds_handle *h, const pqp_collision_in *in, bool mapped, const int32_t *map_index,
                    const pqp_collision_out *out, std::optional<cudaStream_t> stream) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || !in->poses || !in->n || !out->first_hit)
        return fail(h->err, PQP_E_INVALID, "pqp_bounds_collision_check: null in, out, poses, n or first_hit");
    if (in->batch <= 0 || in->n_max <= 0 || in->row_stride < 3)
        return fail(h->err, PQP_E_INVALID, "pqp_bounds_collision_check: batch, n_max > 0 and row_stride >= 3 required");
    if (mapped && !map_index)
        return fail(h->err, PQP_E_INVALID,
                    stream ? "pqp_bounds_collision_check_mapped_device: null map_index"
                           : "pqp_bounds_collision_check_mapped: null map_index");
    pqp::DeviceGuard guard_(h->device);
    if (stream) return launch_collision(h, in, map_index, out, *stream);
    // the extent the kernel reads: rows 0 .. 2 of the last path, so states + n_max needs no padding row
    const size_t B = in->batch, np = ((B - 1) * in->row_stride + 3) * in->n_max, ns = B * in->n_max;
    PQP_CUDA(h->err, h->res.grow(h->d_states, np));
    PQP_CUDA(h->err, h->res.grow(h->d_n, B));
    PQP_CUDA(h->err, h->res.grow(h->d_hit, B));
    if (out->state_free) PQP_CUDA(h->err, h->res.grow(h->d_free, ns));
    if (out->clearance) PQP_CUDA(h->err, h->res.grow(h->d_clear, ns));
    if (mapped) PQP_CUDA(h->err, h->res.grow(h->d_map_index, B));
    cudaStream_t s = h->stream;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_states, in->poses, np * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_n, in->n, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    if (mapped)
        PQP_CUDA(h->err, cudaMemcpyAsync(h->d_map_index, map_index, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    pqp_collision_in din = *in;
    din.poses = h->d_states;
    din.n = h->d_n;
    const pqp_collision_out dout = {h->d_hit, out->state_free ? h->d_free : nullptr,
                                    out->clearance ? h->d_clear : nullptr};
    const int rc = launch_collision(h, &din, mapped ? h->d_map_index : nullptr, &dout, s);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(h->err, cudaMemcpyAsync(out->first_hit, h->d_hit, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (out->state_free)
        PQP_CUDA(h->err, cudaMemcpyAsync(out->state_free, h->d_free, ns, cudaMemcpyDeviceToHost, s));
    if (out->clearance)
        PQP_CUDA(h->err, cudaMemcpyAsync(out->clearance, h->d_clear, ns * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaStreamSynchronize(s));
    return PQP_OK;
}

}  // namespace

extern "C" {

void pqp_bounds_default_params(pqp_bounds_params *p) {
    if (!p) return;
    p->front_length = 3.9;
    p->rear_length = -1.0;
    p->car_width = 2.0;
    p->safety_margin = 0.3;
    p->epsilon = 1e-6;
}

int pqp_bounds_create(const pqp_bounds_map *map, const pqp_bounds_params *params, int32_t device,
                      pqp_bounds_handle **out) {
    return create(map, 1, params, device, out, "pqp_bounds_create");
}

int pqp_bounds_create_maps(const pqp_bounds_map *maps, int32_t n_maps, const pqp_bounds_params *params,
                           int32_t device, pqp_bounds_handle **out) {
    return create(maps, n_maps, params, device, out, "pqp_bounds_create_maps");
}

void pqp_bounds_destroy(pqp_bounds_handle *h) {
    delete h;
}

int32_t pqp_bounds_map_count(const pqp_bounds_handle *h) { return h ? h->n_maps : 0; }

int pqp_bounds_compute_device(pqp_bounds_handle *h, const pqp_bounds_in *in, const pqp_bounds_out *out, void *stream) {
    return compute(h, in, false, nullptr, out, static_cast<cudaStream_t>(stream));
}

int pqp_bounds_compute(pqp_bounds_handle *h, const pqp_bounds_in *in, const pqp_bounds_out *out) {
    return compute(h, in, false, nullptr, out, std::nullopt);
}

int pqp_bounds_compute_mapped_device(pqp_bounds_handle *h, const pqp_bounds_in *in, const int32_t *map_index,
                                     const pqp_bounds_out *out, void *stream) {
    return compute(h, in, true, map_index, out, static_cast<cudaStream_t>(stream));
}

int pqp_bounds_compute_mapped(pqp_bounds_handle *h, const pqp_bounds_in *in, const int32_t *map_index,
                              const pqp_bounds_out *out) {
    return compute(h, in, true, map_index, out, std::nullopt);
}

int pqp_bounds_collision_check(pqp_bounds_handle *h, const pqp_collision_in *in, const pqp_collision_out *out) {
    return collision_check(h, in, false, nullptr, out, std::nullopt);
}

int pqp_bounds_collision_check_device(pqp_bounds_handle *h, const pqp_collision_in *in, const pqp_collision_out *out,
                                      void *stream) {
    return collision_check(h, in, false, nullptr, out, static_cast<cudaStream_t>(stream));
}

int pqp_bounds_collision_check_mapped(pqp_bounds_handle *h, const pqp_collision_in *in, const int32_t *map_index,
                                      const pqp_collision_out *out) {
    return collision_check(h, in, true, map_index, out, std::nullopt);
}

int pqp_bounds_collision_check_mapped_device(pqp_bounds_handle *h, const pqp_collision_in *in,
                                             const int32_t *map_index, const pqp_collision_out *out, void *stream) {
    return collision_check(h, in, true, map_index, out, static_cast<cudaStream_t>(stream));
}

static int validate_states(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out || in->batch <= 0 || in->n_max <= 0 || in->k_max < 3 || !in->spline || !in->k || !in->max_s ||
        !out->states || !out->curvature || !out->n || !(in->delta_s_larger > 0.0) || !(in->delta_s_smaller > 0.0) ||
        in->delta_s_smaller > in->delta_s_larger)
        return fail(h->err, PQP_E_INVALID,
                    "pqp_bounds_build_states: null pointer, non-positive size, or 0 < delta_s_smaller <= delta_s_larger violated");
    return PQP_OK;
}

static int launch_states(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out, cudaStream_t s) {
    StatesArgs a;
    a.batch = in->batch;
    a.n_max = in->n_max;
    a.k_max = in->k_max;
    a.spline = in->spline;
    a.k = in->k;
    a.max_s = in->max_s;
    a.ds_small = in->delta_s_smaller;
    a.ds_large = in->delta_s_larger;
    a.dynamic = in->dynamic_segmentation;
    a.states = out->states;
    a.curvature = out->curvature;
    a.knots = out->knots;
    a.n = out->n;
    a.total = out->total;
    PQP_CUDA(h->err, cudaEventRecord(h->ev0, s));
    reference_states_kernel<<<(in->batch + 63) / 64, 64, 0, s>>>(a);
    PQP_CUDA(h->err, cudaGetLastError());
    PQP_CUDA(h->err, cudaEventRecord(h->ev1, s));
    h->timed = true;
    return PQP_OK;
}

// pqp_bounds_build_states(_device); `stream` empty: the host form, as compute's
static int build_states(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out,
                        std::optional<cudaStream_t> stream) {
    int rc = validate_states(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    if (stream) return launch_states(h, in, out, *stream);
    const size_t B = in->batch, ns = B * PQP_STATE_ROWS * in->n_max, nsp = B * PQP_SPLINE_ROWS * in->k_max;
    const size_t nc = B * in->n_max, nk = out->knots ? B * PQP_NFIELDS * in->n_max : 0;
    PQP_CUDA(h->err, h->res.grow(h->d_states, ns));
    PQP_CUDA(h->err, h->res.grow(h->d_curv, nc));
    PQP_CUDA(h->err, h->res.grow(h->d_spline, nsp));
    if (nk) PQP_CUDA(h->err, h->res.grow(h->d_knots, nk));
    PQP_CUDA(h->err, h->res.grow(h->d_n, B));
    PQP_CUDA(h->err, h->res.grow(h->d_k, B));
    PQP_CUDA(h->err, h->res.grow(h->d_total, B));
    PQP_CUDA(h->err, h->res.grow(h->d_maxs, B));
    cudaStream_t s = h->stream;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_spline, in->spline, nsp * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_k, in->k, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->d_maxs, in->max_s, B * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_states, 0, ns * sizeof(double), s));
    PQP_CUDA(h->err, cudaMemsetAsync(h->d_curv, 0, nc * sizeof(double), s));
    if (nk) PQP_CUDA(h->err, cudaMemcpyAsync(h->d_knots, out->knots, nk * sizeof(double), cudaMemcpyHostToDevice, s));
    pqp_states_in din = *in;
    din.spline = h->d_spline;
    din.k = h->d_k;
    din.max_s = h->d_maxs;
    pqp_states_out dout;
    dout.states = h->d_states;
    dout.curvature = h->d_curv;
    dout.n = h->d_n;
    dout.total = h->d_total;
    dout.knots = nk ? h->d_knots : nullptr;
    rc = launch_states(h, &din, &dout, s);
    if (rc != PQP_OK) return rc;
    PQP_CUDA(h->err, cudaMemcpyAsync(out->states, h->d_states, ns * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->curvature, h->d_curv, nc * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->n, h->d_n, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (out->total) PQP_CUDA(h->err, cudaMemcpyAsync(out->total, h->d_total, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (nk) PQP_CUDA(h->err, cudaMemcpyAsync(out->knots, h->d_knots, nk * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaStreamSynchronize(s));
    return PQP_OK;
}

int pqp_bounds_build_states_device(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out, void *stream) {
    return build_states(h, in, out, static_cast<cudaStream_t>(stream));
}

int pqp_bounds_build_states(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out) {
    return build_states(h, in, out, std::nullopt);
}

int pqp_bounds_last_kernel_ms(pqp_bounds_handle *h, float *ms) {
    if (!h || !ms) return PQP_E_INVALID;
    if (!h->timed) {
        *ms = 0.0f;
        return PQP_OK;
    }
    PQP_CUDA(h->err, cudaEventSynchronize(h->ev1));
    PQP_CUDA(h->err, cudaEventElapsedTime(ms, h->ev0, h->ev1));
    return PQP_OK;
}

const char *pqp_bounds_last_error(pqp_bounds_handle *h) { return h ? h->err.c_str() : g_bounds_create_error.c_str(); }

int pqp_bounds_set_map_device(pqp_bounds_handle *h, const pqp_bounds_map *map, void *stream) {
    return set_map_slot(h, 0, map, static_cast<cudaStream_t>(stream), "pqp_bounds_set_map");
}

int pqp_bounds_set_map(pqp_bounds_handle *h, const pqp_bounds_map *map) {
    return set_map_slot(h, 0, map, std::nullopt, "pqp_bounds_set_map");
}

int pqp_bounds_set_map_slot_device(pqp_bounds_handle *h, int32_t slot, const pqp_bounds_map *map, void *stream) {
    return set_map_slot(h, slot, map, static_cast<cudaStream_t>(stream), "pqp_bounds_set_map_slot");
}

int pqp_bounds_set_map_slot(pqp_bounds_handle *h, int32_t slot, const pqp_bounds_map *map) {
    return set_map_slot(h, slot, map, std::nullopt, "pqp_bounds_set_map_slot");
}

int pqp_bounds_set_occupancy_device(pqp_bounds_handle *h, const pqp_occupancy_map *occ, void *stream) {
    return occupancy_image(h, occ, static_cast<cudaStream_t>(stream), "pqp_bounds_set_occupancy_device");
}

int pqp_bounds_set_occupancy(pqp_bounds_handle *h, const pqp_occupancy_map *occ) {
    return occupancy_image(h, occ, std::nullopt, "pqp_bounds_set_occupancy");
}

int pqp_bounds_set_occupancy_slots_device(pqp_bounds_handle *h, int32_t first_slot, const pqp_occupancy_stack *stack,
                                          void *stream) {
    return occupancy(h, {first_slot, stack, false, 0, nullptr, false}, static_cast<cudaStream_t>(stream),
                     "pqp_bounds_set_occupancy_slots_device");
}

int pqp_bounds_set_occupancy_slots(pqp_bounds_handle *h, int32_t first_slot, const pqp_occupancy_stack *stack) {
    return occupancy(h, {first_slot, stack, false, 0, nullptr, false}, std::nullopt, "pqp_bounds_set_occupancy_slots");
}

int pqp_bounds_set_occupancy_boxes_device(pqp_bounds_handle *h, int32_t first_slot, const pqp_occupancy_stack *base,
                                          int32_t shared_base, const pqp_obstacle_boxes *boxes, void *stream) {
    return occupancy(h, {first_slot, base, true, shared_base, boxes, false}, static_cast<cudaStream_t>(stream),
                     "pqp_bounds_set_occupancy_boxes_device");
}

int pqp_bounds_set_occupancy_boxes(pqp_bounds_handle *h, int32_t first_slot, const pqp_occupancy_stack *base,
                                   int32_t shared_base, const pqp_obstacle_boxes *boxes) {
    return occupancy(h, {first_slot, base, true, shared_base, boxes, false}, std::nullopt,
                     "pqp_bounds_set_occupancy_boxes");
}

int pqp_bounds_get_map(pqp_bounds_handle *h, pqp_bounds_map *meta, float *distance) {
    return get_map_slot(h, 0, meta, distance, "pqp_bounds_get_map");
}

int pqp_bounds_get_map_slot(pqp_bounds_handle *h, int32_t slot, pqp_bounds_map *meta, float *distance) {
    return get_map_slot(h, slot, meta, distance, "pqp_bounds_get_map_slot");
}

}  // extern "C"
