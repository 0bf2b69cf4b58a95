// test_comm_ranks.cpp -- drives N ranks (one process each) through include/sprs_b200.h ONLY:
// rendezvous by id, nnz-balanced row partition, symmetric y / x buffers, the row-partitioned
// SpMV in every exchange mode (device-resident and host-vector forms), device barrier.
// The ranks use device rank % n_devices, so on a single-GPU box both ranks share device 0 and
// the whole multi-rank logic still runs on hardware.  Usage: test_comm_ranks [world]
// Checks: every rank ends with the FULL y = A x for every exchange mode, twice in a row with a
// different x each time, BIT FOR BIT against the sequential CPU sum of this file.  A and x hold
// small integers, so every partial sum is exact and every summation order gives the same bits;
// a row that is dropped, doubled, misplaced or left over from the previous product fails.
#include <sys/wait.h>
#include <unistd.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/sprs_b200.h"

#define CK(ctx, call)                                                                          \
    do {                                                                                       \
        int _s = (call);                                                                       \
        if (_s != SPRS_B200_OK) {                                                              \
            fprintf(stderr, "[rank %d] %s -> %d: %s (%s:%d)\n", g_rank, #call, _s,             \
                    sprs_b200_last_error(ctx), __FILE__, __LINE__);                            \
            exit(2);                                                                           \
        }                                                                                      \
    } while (0)

static int g_rank = -1;

static uint64_t splitmix(uint64_t& s) {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
// a non-zero integer in [-m, m]: |A| <= 8, |x| <= 1024 and rows of at most 5000 non-zeros keep
// every partial sum below 2^26, far inside the exact range of a double
static double small_int(uint64_t& s, uint64_t m) {
    const uint64_t h = splitmix(s);
    return (double)(h % m + 1) * ((h >> 32) & 1 ? -1.0 : 1.0);
}
static bool same_bits(double a, double b) { return memcmp(&a, &b, sizeof a) == 0; }

struct Csr {
    uint64_t rows, cols;
    std::vector<uint32_t> indptr, indices;
    std::vector<double> data;
};

// skewed test matrix: empty rows, short rows and a few hubs, ascending unique columns
static Csr make_matrix(uint64_t rows, uint64_t cols, uint64_t seed) {
    Csr m{rows, cols, {0}, {}, {}};
    uint64_t s = seed;
    for (uint64_t r = 0; r < rows; ++r) {
        uint64_t len = splitmix(s) % 40;
        if (r % 11 == 0) len = 0;
        if (r % 997 == 5) len = 3000 + splitmix(s) % 2000;
        if (len > cols) len = cols;
        uint64_t c = splitmix(s) % (cols / (len + 1) + 1);
        for (uint64_t k = 0; k < len && c < cols; ++k) {
            m.indices.push_back((uint32_t)c);
            m.data.push_back(small_int(s, 8));
            c += 1 + splitmix(s) % (2 * cols / (len + 1) + 1) / 2;
        }
        m.indptr.push_back((uint32_t)m.indices.size());
    }
    return m;
}

static int run_rank(int rank, int world, const char* id) {
    g_rank = rank;
    int ndev = 1;
    const char* nd = getenv("SPRS_TEST_NDEV");
    if (nd) ndev = atoi(nd);
    sprs_b200_ctx* ctx = nullptr;
    if (sprs_b200_ctx_create(rank % ndev, &ctx) != SPRS_B200_OK) {
        fprintf(stderr, "[rank %d] ctx_create: %s\n", rank, sprs_b200_last_error(nullptr));
        return 3;
    }
    sprs_b200_comm* comm = nullptr;
    CK(ctx, sprs_b200_comm_init_rank(ctx, id, rank, world, &comm));
    if (sprs_b200_comm_rank(comm) != rank || sprs_b200_comm_world(comm) != world) return 4;

    const uint64_t n = 20000;
    const Csr a = make_matrix(n, n, 0x5EED);
    // two x vectors used in turn, so that a stale row of the previous product is wrong
    std::vector<double> xv[2] = {std::vector<double>(n), std::vector<double>(n)};
    std::vector<double> ref[2] = {std::vector<double>(n, 0.0), std::vector<double>(n, 0.0)};
    uint64_t s = 77;
    for (int v = 0; v < 2; ++v) {
        for (auto& e : xv[v]) e = small_int(s, 1024);
        for (uint64_t r = 0; r < n; ++r)
            for (uint32_t k = a.indptr[r]; k < a.indptr[r + 1]; ++k)
                ref[v][r] += a.data[k] * xv[v][a.indices[k]];
    }
    // partition (every rank computes the same cut points) and this rank's block
    std::vector<uint64_t> bounds(world + 1);
    CK(ctx, sprs_b200_partition_rows(a.indptr.data(), 4, n, world, 8.0, bounds.data()));
    if (bounds[0] != 0 || bounds[world] != n) return 5;
    for (int g = 0; g < world; ++g)
        if (bounds[g] > bounds[g + 1]) return 5;
    const uint64_t r0 = bounds[rank], r1 = bounds[rank + 1];
    // this rank's block = slice_outer(r0..r1): the indptr slice is NOT zero-based (upload
    // rebases it, like proper_indptr), indices / data start at the block's first non-zero
    sprs_b200_csmat* blk = nullptr;
    CK(ctx, sprs_b200_csmat_upload(ctx, SPRS_B200_CSR, r1 - r0, n, a.indptr.data() + r0, 4,
                                   a.indices.data() + a.indptr[r0], 4, a.data.data() + a.indptr[r0],
                                   &blk));
    // small all-gather through the communicator: every rank's block nnz
    uint64_t my_nnz = sprs_b200_csmat_nnz(blk), all_nnz[SPRS_B200_MAX_RANKS] = {};
    CK(ctx, sprs_b200_comm_allgather_host(comm, &my_nnz, 8, all_nnz));
    uint64_t tot = 0;
    for (int g = 0; g < world; ++g) tot += all_nnz[g];
    if (tot != a.indices.size()) return 6;

    // a mismatch is reported and remembered, never returned early: the other ranks wait for this
    // one at every collective call below, so it keeps making them
    int checks = 0, fail = 0;
    for (int want_mc = 0; want_mc <= 1; ++want_mc) {
        sprs_b200_symm *y = nullptr, *xs = nullptr;
        CK(ctx, sprs_b200_symm_alloc(comm, n * 8, want_mc, &y));
        CK(ctx, sprs_b200_symm_alloc(comm, n * 8, want_mc, &xs));
        const bool mc = sprs_b200_symm_multicast_ptr(y) != nullptr;
        if (want_mc && !mc && rank == 0)
            printf("note: no multicast on this box (supported=%d): unicast peers used\n",
                   sprs_b200_comm_multicast_supported(comm));
        // device-resident form: x replicated, y all-gathered
        double* d_x = (double*)sprs_b200_symm_ptr(xs, rank);
        for (int mode : {SPRS_B200_EXCHANGE_FUSED, SPRS_B200_EXCHANGE_PUSH, SPRS_B200_EXCHANGE_AUTO}) {
            for (int rep = 0; rep < 2; ++rep) {
                // the host-vector form uploads this rep's x (also tests the x all-gather); the
                // device-resident form below then reads the same x from the symmetric buffer
                std::vector<double> yh(r1 - r0, NAN);
                CK(ctx, sprs_b200_mul_mat_vec_rowpart(comm, blk, xs, xv[rep].data() + r0, r0, r1 - r0,
                                                      yh.data(), r1 - r0));
                for (uint64_t r = r0; r < r1; ++r, ++checks)
                    if (!same_bits(yh[r - r0], ref[rep][r])) {
                        fprintf(stderr, "[rank %d] e2e mc=%d rep %d row %llu: %.17g vs %.17g\n", rank,
                                (int)mc, rep, (unsigned long long)r, yh[r - r0], ref[rep][r]);
                        fail = 7;
                        break;
                    }
                // poison this rank's y so that a row that never arrives is caught
                std::vector<double> poison(n, NAN), got(n);
                CK(ctx, sprs_b200_comm_barrier_dev(comm, nullptr));
                CK(ctx, sprs_b200_comm_check(comm, nullptr));
                CK(ctx, sprs_b200_copy_to_device(ctx, sprs_b200_symm_ptr(y, rank), poison.data(), n * 8, nullptr));
                CK(ctx, sprs_b200_comm_barrier_dev(comm, nullptr));
                CK(ctx, sprs_b200_spmv_rowpart(comm, blk, d_x, y, r0, mode, nullptr));
                CK(ctx, sprs_b200_comm_check(comm, nullptr));
                CK(ctx, sprs_b200_copy_to_host(ctx, got.data(), sprs_b200_symm_ptr(y, rank), n * 8, nullptr));
                for (uint64_t r = 0; r < n; ++r, ++checks)
                    if (!same_bits(got[r], ref[rep][r])) {
                        fprintf(stderr, "[rank %d] mode %d mc=%d rep %d row %llu: %.17g vs %.17g\n", rank,
                                mode, (int)mc, rep, (unsigned long long)r, got[r], ref[rep][r]);
                        fail = 9;
                        break;
                    }
            }
        }
        CK(ctx, sprs_b200_symm_free(xs));
        CK(ctx, sprs_b200_symm_free(y));
    }
    sprs_b200_csmat_free(blk);
    CK(ctx, sprs_b200_comm_free(comm));
    sprs_b200_ctx_destroy(ctx);
    if (fail) return fail;
    if (rank == 0) printf("OK %d checks per rank, world %d\n", checks, world);
    return 0;
}

int main(int argc, char** argv) {
    const int world = argc > 1 ? atoi(argv[1]) : 2;
    if (argc > 3) return run_rank(atoi(argv[2]), world, argv[3]);  // child: rank, id
    if (world < 1 || world > SPRS_B200_MAX_RANKS) return 1;
    char id[64];
    if (sprs_b200_comm_unique_id(id) != SPRS_B200_OK) return 1;
    std::vector<pid_t> kids;
    for (int r = 0; r < world; ++r) {
        pid_t p = fork();  // the parent never touches CUDA, so fork + exec is safe
        if (p == 0) {
            const std::string rs = std::to_string(r), ws = std::to_string(world);
            execl(argv[0], argv[0], ws.c_str(), rs.c_str(), id, (char*)nullptr);
            _exit(127);
        }
        kids.push_back(p);
    }
    int bad = 0;
    for (pid_t p : kids) {
        int st = 0;
        waitpid(p, &st, 0);
        if (!WIFEXITED(st) || WEXITSTATUS(st) != 0) {
            fprintf(stderr, "rank process %d: status %d\n", (int)p, WIFEXITED(st) ? WEXITSTATUS(st) : -1);
            bad = 1;
        }
    }
    return bad;
}
