// batch_layout_test.cpp — TEST ONLY, host code (g++). The batch table of pqp_batch_layout.h against the element
// counts the solver's host calls used per member before the table existed, written out member by member, and
// batch_from's offsets. Prints "ok <in members> <out members>" or the first mismatch and exits non-zero.
#include <cstdio>

#include "../../path_optimizer_2_b200/csrc/pqp_batch_layout.h"

namespace {

int fails = 0;

void expect(const char *what, size_t got, size_t want) {
    if (got != want && fails++ < 10) std::printf("mismatch %s: %zu per instance, expected %zu\n", what, got, want);
}

}  // namespace

int main() {
    const size_t N = 239, d = sizeof(double), i4 = sizeof(int32_t);
    const auto fi = pqp::batch_fields((const pqp_batch_in *)nullptr, N);
    const auto fo = pqp::batch_fields((const pqp_batch_out *)nullptr, N);
    size_t at = 0;
    // the expected elements and element size of one member, in the table's order (a missing or reordered member
    // fails here); per_instance must find the same count
#define CHECK(table, type, member, elems, elem_bytes)                                               \
    do {                                                                                            \
        if (at >= table.size() || table[at].offset != offsetof(type, member)) {                     \
            std::printf("mismatch %s: not field %zu of the table\n", #member, at);                \
            return 1;                                                                               \
        }                                                                                           \
        expect(#member, table[at].count, (elems));                                                  \
        expect(#member " element bytes", table[at++].size, (elem_bytes));                           \
        expect(#member " per_instance", pqp::per_instance(&type::member, N), (elems));             \
    } while (0)
    CHECK(fi, pqp_batch_in, knots, PQP_NFIELDS * N, d);
    CHECK(fi, pqp_batch_in, inst, PQP_NINST, d);
    CHECK(fi, pqp_batch_in, n, 1, i4);
    CHECK(fi, pqp_batch_in, p, 1, i4);
    if (at != fi.size()) {
        std::printf("mismatch: %zu pqp_batch_in members checked, the table has %zu\n", at, fi.size());
        return 1;
    }
    at = 0;
    // the order the host calls copied the outputs in: info before the full outputs
    CHECK(fo, pqp_batch_out, sol, 4 * N, d);
    CHECK(fo, pqp_batch_out, cost, 1, d);
    CHECK(fo, pqp_batch_out, status, 1, i4);
    CHECK(fo, pqp_batch_out, iters, 1, i4);
    CHECK(fo, pqp_batch_out, info, PQP_NINFO, d);
    CHECK(fo, pqp_batch_out, x_full, 6 * N - 1, d);
    CHECK(fo, pqp_batch_out, y_full, 6 * N + 2, d);
    CHECK(fo, pqp_batch_out, z_full, 6 * N + 2, d);
#undef CHECK
    if (at != fo.size()) {
        std::printf("mismatch: %zu pqp_batch_out members checked, the table has %zu\n", at, fo.size());
        return 1;
    }
    // every pointer member is in the table
    if (fi.size() != (sizeof(pqp_batch_in) - 2 * sizeof(int32_t)) / sizeof(void *) ||
        fo.size() != sizeof(pqp_batch_out) / sizeof(void *)) {
        std::printf("mismatch: a pointer member is missing from the table\n");
        return 1;
    }
    // batch_from: a set member moves by first * its elements per instance, a NULL one stays NULL
    static double knots[16 * PQP_NFIELDS * N], y_full[16 * (6 * N + 2)];
    static int32_t n[16], status[16];
    const pqp_batch_in in = {16, (int32_t)N, knots, nullptr, n, nullptr};
    const pqp_batch_in vi = pqp::batch_from(in, 5, N);
    if (vi.batch != 16 || vi.n_max != (int32_t)N || vi.knots != knots + 5 * PQP_NFIELDS * N || vi.inst != nullptr ||
        vi.n != n + 5 || vi.p != nullptr) {
        std::printf("mismatch: batch_from offsets of pqp_batch_in\n");
        return 1;
    }
    pqp_batch_out out{};
    out.status = status;
    out.y_full = y_full;
    const pqp_batch_out vo = pqp::batch_from(out, 7, N);
    if (vo.status != status + 7 || vo.y_full != y_full + 7 * (6 * N + 2) || vo.sol != nullptr || vo.cost != nullptr ||
        vo.iters != nullptr || vo.x_full != nullptr || vo.z_full != nullptr || vo.info != nullptr) {
        std::printf("mismatch: batch_from offsets of pqp_batch_out\n");
        return 1;
    }
    if (fails) return 1;
    std::printf("ok %zu %zu\n", fi.size(), fo.size());
    return 0;
}
