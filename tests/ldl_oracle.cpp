// ldl_oracle.cpp -- TEST INFRASTRUCTURE ONLY: a restatement of the sprs-ldl crate's
// ldl_symbolic, ldl_numeric (its early return included), ldl_lsolve, ldl_ltsolve, of
// sprs::linalg::diag_solve and of the permutation product `&perm * v`, that the device
// factorization (csrc/ldl.cu) is compared with bit for bit.  The numeric pattern is built with
// the reference's two-sided stack (sprs::stack::DStack) as it is used there, so the order of
// every subtraction follows from the stack, not from a description of it.  Built with
// -ffp-contract=off (no FMA, like sprs) by tests/ldl_oracle.py.
//
// Arrays: indptr u64 (zero-based), indices u32 ascending per outer dimension, f64 data; perm and
// pinv u64 (perm[k] = the outer vector that is row k; pinv its inverse).  L is CSC: colptr u64,
// row indices u64.
#include <cstdint>
#include <vector>

namespace {

constexpr uint64_t NONE = ~0ull;

// sprs::stack::DStack: a left stack growing up from 0 and a right stack growing down from n
struct DStack {
    std::vector<uint64_t> stacks;
    int64_t left_head = -1;
    uint64_t right_head;
    explicit DStack(uint64_t n) : stacks(n), right_head(n) {}
    void push_left(uint64_t v) { stacks[++left_head] = v; }
    void push_right(uint64_t v) { stacks[--right_head] = v; }
    bool pop_left(uint64_t* v) {
        if (left_head < 0) return false;
        *v = stacks[left_head--];
        return true;
    }
    void clear_left() { left_head = -1; }
    void clear_right() { right_head = stacks.size(); }
    void push_left_on_right() {
        uint64_t v;
        while (pop_left(&v)) push_right(v);
    }
};

}  // namespace

extern "C" {

// ldl_symbolic: the elimination tree (parent, NONE for a root), the column counts l_nz and
// colptr (n + 1 entries).  flag: n entries of workspace, left as the reference leaves it.
void oracle_ldl_symbolic(uint64_t n, const uint64_t* ip, const uint32_t* idx, const uint64_t* perm,
                         const uint64_t* pinv, uint64_t* colptr, uint64_t* parent, uint64_t* l_nz,
                         uint64_t* flag) {
    for (uint64_t k = 0; k < n; ++k) {
        const uint64_t o = perm[k];
        flag[k] = k;
        parent[k] = NONE;
        l_nz[k] = 0;
        for (uint64_t p = ip[o]; p < ip[o + 1]; ++p) {
            uint64_t i = pinv[idx[p]];
            if (i < k) {
                while (flag[i] != k) {
                    if (parent[i] == NONE) parent[i] = k;  // uproot
                    l_nz[i] += 1;
                    flag[i] = k;
                    i = parent[i];
                }
            }
        }
    }
    uint64_t prev = 0;
    for (uint64_t k = 0; k < n; ++k) {
        colptr[k] = prev;
        prev += l_nz[k];
    }
    colptr[n] = prev;
}

// ldl_numeric: L's row indices and values (colptr[n] entries), D.  l_nz, y (n entries, zero on
// the first call) and flag are the reference's workspaces and carry over between calls as
// there.  Returns 0 for Ok, else 1 + the index of the SingularMatrix.
uint64_t oracle_ldl_numeric(uint64_t n, const uint64_t* ip, const uint32_t* idx, const double* val,
                            const uint64_t* perm, const uint64_t* pinv, const uint64_t* colptr,
                            const uint64_t* parent, uint64_t* l_nz, uint64_t* l_idx,
                            double* l_val, double* diag, double* y, uint64_t* flag) {
    DStack pattern(n);
    for (uint64_t k = 0; k < n; ++k) {
        const uint64_t o = perm[k];
        flag[k] = k;
        y[k] = 0.0;
        l_nz[k] = 0;
        pattern.clear_right();
        for (uint64_t p = ip[o]; p < ip[o + 1]; ++p) {
            const uint64_t inner = pinv[idx[p]];
            if (inner > k) continue;
            y[inner] = y[inner] + val[p];
            uint64_t i = inner;
            pattern.clear_left();
            while (flag[i] != k) {
                pattern.push_left(i);
                flag[i] = k;
                i = parent[i];
            }
            pattern.push_left_on_right();
        }
        diag[k] = y[k];
        y[k] = 0.0;
        for (uint64_t q = pattern.right_head; q < n; ++q) {
            const uint64_t i = pattern.stacks[q];
            const double yi = y[i];
            y[i] = 0.0;
            const uint64_t p2 = colptr[i] + l_nz[i];
            for (uint64_t p = colptr[i]; p < p2; ++p) y[l_idx[p]] = y[l_idx[p]] - l_val[p] * yi;
            const double l_ki = yi / diag[i];
            diag[k] = diag[k] - l_ki * yi;
            l_idx[p2] = k;
            l_val[p2] = l_ki;
            l_nz[i] += 1;
        }
        if (diag[k] == 0.0) return 1 + k;
    }
    return 0;
}

// ldl_lsolve: the column sweep of the unit lower L (CSC)
void oracle_ldl_lsolve(uint64_t n, const uint64_t* colptr, const uint64_t* l_idx,
                       const double* l_val, double* x) {
    for (uint64_t c = 0; c < n; ++c) {
        const double xc = x[c];
        for (uint64_t p = colptr[c]; p < colptr[c + 1]; ++p) x[l_idx[p]] -= l_val[p] * xc;
    }
}

// ldl_ltsolve: L^T x = b, columns of L in descending order
void oracle_ldl_ltsolve(uint64_t n, const uint64_t* colptr, const uint64_t* l_idx,
                        const double* l_val, double* x) {
    for (uint64_t c = n; c-- > 0;) {
        double xo = x[c];
        for (uint64_t p = colptr[c]; p < colptr[c + 1]; ++p) xo -= l_val[p] * x[l_idx[p]];
        x[c] = xo;
    }
}

// linalg::diag_solve
void oracle_diag_solve(uint64_t n, const double* d, double* x) {
    for (uint64_t i = 0; i < n; ++i) x[i] /= d[i];
}

// `&perm * v`: out[i] = v[perm[i]]
void oracle_perm_mul(uint64_t n, const uint64_t* perm, const double* v, double* out) {
    for (uint64_t i = 0; i < n; ++i) out[i] = v[perm[i]];
}

// Height of the elimination tree (for reports): the number of nodes on its longest
// leaf-to-root path (0 for n == 0).  parent[i] > i or NONE.
uint64_t oracle_etree_height(uint64_t n, const uint64_t* parent, uint64_t* depth) {
    uint64_t h = 0;
    for (uint64_t i = n; i-- > 0;) {
        depth[i] = parent[i] == NONE ? 1 : depth[parent[i]] + 1;
        if (depth[i] > h) h = depth[i];
    }
    return h;
}

}  // extern "C"
