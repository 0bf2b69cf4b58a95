// construct_oracle.cpp -- TEST INFRASTRUCTURE ONLY: the CPU restatement of sprs's matrix
// construction that the device results are compared with bit for bit (tests/construct_oracle.py
// loads it and restates the composition of bmat / vstack / hstack on top of these).
//
//   oracle_convert   to_other_storage (raw::convert_mat_storage, csmat.rs:1782-1829): a counting
//                    transpose -- count the entries of every inner index, scan, then place each
//                    outer vector's entries in order, so that indices come out ascending.
//   oracle_stack     same_storage_fast_stack (construct.rs): the outer vectors of every matrix
//                    appended one after the other (append_outer_csvec), values copied.
//   oracle_kron      kronecker_product (kronecker.rs), its double loop: for each outer vector
//                    of a, each outer vector of b, each entry of a's, each entry of b's:
//                    index ja * inner(b) + jb, value va * vb.
//
// Everything is u64 indptr / u64 indices and indptr arrays are zero-based.  Single-threaded,
// like the reference.  -ffp-contract=off.
#include <cstddef>
#include <cstdint>
#include <vector>

extern "C" void oracle_convert(uint64_t outer, uint64_t inner, const uint64_t* ip,
                               const uint64_t* ind, const double* dat, uint64_t* out_ip,
                               uint64_t* out_ind, double* out_dat) {
    std::vector<uint64_t> count(inner + 1, 0);
    for (uint64_t k = 0; k < ip[outer]; ++k) ++count[ind[k] + 1];
    for (uint64_t i = 0; i < inner; ++i) count[i + 1] += count[i];
    for (uint64_t i = 0; i <= inner; ++i) out_ip[i] = count[i];
    for (uint64_t o = 0; o < outer; ++o)
        for (uint64_t k = ip[o]; k < ip[o + 1]; ++k) {
            const uint64_t dst = count[ind[k]]++;
            out_ind[dst] = o;
            out_dat[dst] = dat[k];
        }
}

// n matrices, their indptrs concatenated (outers[m] + 1 entries each), indices and data
// concatenated; the result's indptr has sum(outers) + 1 entries
extern "C" void oracle_stack(uint64_t n, const uint64_t* outers, const uint64_t* ips,
                             const uint64_t* inds, const double* dats, uint64_t* out_ip,
                             uint64_t* out_ind, double* out_dat) {
    uint64_t nnz = 0, row = 0, src = 0;
    out_ip[0] = 0;
    for (uint64_t m = 0; m < n; ++m) {
        const uint64_t* ip = ips;
        for (uint64_t o = 0; o < outers[m]; ++o) {
            for (uint64_t k = ip[o]; k < ip[o + 1]; ++k) {
                out_ind[nnz] = inds[src + k];
                out_dat[nnz] = dats[src + k];
                ++nnz;
            }
            out_ip[++row] = nnz;
        }
        src += ip[outers[m]];
        ips += outers[m] + 1;
    }
}

extern "C" void oracle_kron(uint64_t outer_a, const uint64_t* ipa, const uint64_t* inda,
                            const double* data, uint64_t outer_b, uint64_t inner_b,
                            const uint64_t* ipb, const uint64_t* indb, const double* datb,
                            uint64_t* out_ip, uint64_t* out_ind, double* out_dat) {
    uint64_t count = 0, row = 0;
    out_ip[0] = 0;
    for (uint64_t oa = 0; oa < outer_a; ++oa) {
        for (uint64_t ob = 0; ob < outer_b; ++ob) {
            for (uint64_t ka = ipa[oa]; ka < ipa[oa + 1]; ++ka)
                for (uint64_t kb = ipb[ob]; kb < ipb[ob + 1]; ++kb) {
                    out_ind[count] = inda[ka] * inner_b + indb[kb];
                    out_dat[count] = data[ka] * datb[kb];
                    ++count;
                }
            out_ip[++row] = count;
        }
    }
}
