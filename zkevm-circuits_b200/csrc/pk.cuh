// pk.cuh -- the device-resident proving key (prover.cu) and the stages that build it, shared with the proving-key file codec
// (pk_serde.cu).
#pragma once
#include "common.cuh"
#include "csf.cuh"

struct zkb_pk {
    zkb_ctx *ctx = nullptr;
    zkb::Csf cs;
    zkb::SlotMap sm;
    uint32_t k = 0, ext_k = 0, E = 0, qdeg = 0, chunk = 0, nsets = 0;
    uint64_t n = 0, N = 0;
    zkb::Fr omega, omega_inv, ext_omega, ext_omega_inv, n_inv, N_inv, zeta;
    std::vector<zkb::Fr> t_inv;
    zkb::DevPool pool;
    std::vector<zkb::Fr *> fixed_values, fixed_polys, sigma_values, sigma_polys;
    zkb::Fr *l0_poly = nullptr, *llast_poly = nullptr, *lblind_poly = nullptr, *xid_poly = nullptr, *omega_pows = nullptr;
    zkb_srs *srs = nullptr;       // shared ParamsKZG handle (owned when the pk was made by the legacy zkb_pk_create)
    bool owns_srs = false;
    // coset evaluations of the proof-independent polynomials (fixed, sigma, X, l_0, l_last, l_blind) for every coset part, like
    // upstream's pk.fixed_cosets / permutation cosets / l0 / l_last / l_active_row: [part][slot] -> n elements, null for the other
    // slots; empty when the cache is off
    std::vector<std::vector<zkb::Fr *>> coset_cache;
    ~zkb_pk() {
        if (owns_srs && srs) zkb_srs_destroy(srs);
    }
    // generator zeta * ext_omega^j of coset part j
    zkb::Fr coset_gen(uint32_t j) const { return fp_mul(zeta, fp_pow_u64(ext_omega, j)); }
};

namespace zkb {
// The stages of every pk constructor, in this order on the context's stream: pk_begin (domain, l_0 / l_last / l_blind / X in
// coefficient form), pk_ingest of the fixed and then of the sigma columns (values from host or device pointers -> values and
// coefficient form), pk_finish (the coset cache decision and fill; synchronises).  zkb_pk_read runs the same stages, so a key read from
// a file is the key zkb_pk_create_with_srs builds from the same values.
int32_t pk_begin(zkb_ctx *ctx, Csf &&csf, zkb_srs *srs, zkb_pk **out);
int32_t pk_ingest(zkb_pk *pk, const void *const *src, size_t cnt, std::vector<Fr *> &vals, std::vector<Fr *> &polys);
int32_t pk_finish(zkb_pk *pk);
// the quotient table's proof-independent slots in coefficient form (fixed, sigma, X, l_0, l_last, l_blind), null elsewhere
std::vector<Fr *> pk_quotient_polys(const zkb_pk *pk);
// the vk commitments: commit_lagrange of the fixed, then of the sigma columns (a COLLECTIVE with a communicator); synchronises
int32_t pk_vk_commitments(zkb_pk *pk, std::vector<G1Affine> &out);
}  // namespace zkb
