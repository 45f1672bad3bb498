// transcript.cu -- the framing of every transcript kind (see transcript.cuh) and the host-only entry points that let the CPU
// test-suite pin it against the oracle's transcripts without a device.
#include "transcript.cuh"
#include "keccak.h"

namespace zkb {

// base-field coordinate (canonical limbs, < q) -> scalar-field element (x mod r), Montgomery form: snark-verifier's fe_to_fe
static Fr fq_canonical_to_fr(const Fq &c) {
    uint32_t v[8];
    for (int i = 0; i < 8; ++i) v[i] = c.l[i];
    bool ge = true;
    for (int i = 7; i >= 0; --i) {
        if (v[i] != FrParams::P(i)) { ge = v[i] > FrParams::P(i); break; }
    }
    if (ge) {  // q < 2r: one subtraction suffices
        int64_t br = 0;
        for (int i = 0; i < 8; ++i) { int64_t d = (int64_t)v[i] - FrParams::P(i) + br; v[i] = (uint32_t)d; br = d >> 32; }
    }
    Fr out;
    for (int i = 0; i < 8; ++i) out.l[i] = v[i];
    return fp_from_canonical(out);
}
// 32-byte big-endian image of a canonical field element (EvmTranscript absorbs and writes `to_repr()` reversed)
template <class F>
static void push_be32(std::vector<uint8_t> &dst, const F &canonical) {
    const uint8_t *b = (const uint8_t *)canonical.l;
    for (int i = 31; i >= 0; --i) dst.push_back(b[i]);
}
// Challenge255 squeeze of a Blake2b transcript: absorb the 0x00 prefix, then Fr::from_uniform_bytes of the 64-byte digest,
// (lo + hi * 2^256) mod r, computed with Montgomery multiplications by R^2
static Fr blake2b_challenge255(Blake2b &tr) {
    const uint8_t pre = 0;
    tr.update(&pre, 1);
    uint8_t h[64];
    tr.finalize_copy(h);
    Fr lo, hi;
    memcpy(lo.l, h, 32);
    memcpy(hi.l, h + 32, 32);
    const Fr r2 = Fr::r2();
    return fp_add(fp_mul(lo, r2), fp_mul(fp_mul(hi, r2), r2));
}

void Transcript::common_scalar(const Fr &v) {
    if (kind == CALLER) { callback(vt.common_scalar(vt.user, (const uint64_t *)v.l)); return; }
    if (kind == POSEIDON) { pos.update(v); return; }
    if (kind == EVM) { push_be32(evm_buf, fp_to_canonical(v)); return; }
    const uint8_t pre = 2;
    Fr c = fp_to_canonical(v);
    b2.update(&pre, 1);
    b2.update(c.l, 32);
}
void Transcript::write_scalar(const Fr &v) {
    if (kind == CALLER) { callback(vt.write_scalar(vt.user, (const uint64_t *)v.l)); return; }
    common_scalar(v);
    Fr c = fp_to_canonical(v);
    if (kind == EVM) { push_be32(bytes, c); return; }
    const uint8_t *b = (const uint8_t *)c.l;
    bytes.insert(bytes.end(), b, b + 32);
}
int32_t Transcript::write_point(const G1Affine &p) {
    if (p.is_identity()) { set_error("cannot write points at infinity to the transcript"); return ZKB_ERR_STATE; }
    if (kind == CALLER) {
        const int32_t r = vt.write_point(vt.user, (const uint64_t *)&p);
        if (r) { set_error("the caller's transcript refused a point (callback returned %d)", r); callback(r); return ZKB_ERR_STATE; }
        return ZKB_OK;
    }
    Fq x = fp_to_canonical(p.x), y = fp_to_canonical(p.y);
    if (kind == EVM) {  // absorbed and written uncompressed: x || y, big-endian
        push_be32(evm_buf, x); push_be32(evm_buf, y);
        push_be32(bytes, x); push_be32(bytes, y);
        return ZKB_OK;
    }
    if (kind == POSEIDON) {
        pos.update(fq_canonical_to_fr(x));
        pos.update(fq_canonical_to_fr(y));
    } else {
        const uint8_t pre = 1;
        b2.update(&pre, 1);
        b2.update(x.l, 32);
        b2.update(y.l, 32);
    }
    uint8_t comp[32];
    g1_compress(p, comp);
    bytes.insert(bytes.end(), comp, comp + 32);
    return ZKB_OK;
}
Fr Transcript::squeeze() {
    if (kind == CALLER) {
        Fr c = Fr::zero();
        callback(vt.squeeze_challenge(vt.user, (uint64_t *)c.l));
        return c;
    }
    if (kind == POSEIDON) return pos.squeeze();
    if (kind == EVM) {
        // hash the buffer (plus a 0x01 byte when it holds just the previous digest), keep the digest as the new buffer,
        // challenge = digest as a big-endian integer mod r
        if (evm_buf.size() == 32) evm_buf.push_back(1);
        uint8_t h[32];
        keccak256(evm_buf.data(), evm_buf.size(), h);
        evm_buf.assign(h, h + 32);
        Fr v;
        uint8_t *b = (uint8_t *)v.l;
        for (int i = 0; i < 32; ++i) b[i] = h[31 - i];
        return fp_mul(v, Fr::r2());  // Montgomery multiply reduces any 256-bit value: v * R^2 / R = v R mod r
    }
    return blake2b_challenge255(b2);
}
int32_t Transcript::status() const {
    if (cb_error) { set_error("the caller's transcript callback failed (%d)", cb_error); return ZKB_ERR_STATE; }
    return ZKB_OK;
}

}  // namespace zkb
using namespace zkb;

// ---- host-only transcript primitives (no device needed): let the CPU test-suite pin the hashers of the proving session ----
// absorb n Fr elements (Montgomery) into a fresh Poseidon sponge (PoseidonTranscript::common_scalar) and squeeze one challenge
extern "C" int32_t zkb_poseidon_hash_host(const uint64_t *inputs, uint64_t n, uint64_t out[4]) {
    ZKB_ARG(out && (inputs || n == 0));
    PoseidonSponge sp;
    for (uint64_t i = 0; i < n; ++i) {
        Fr v;
        memcpy(v.l, inputs + 4 * i, 32);
        sp.update(v);
    }
    const Fr c = sp.squeeze();
    memcpy(out, c.l, 32);
    return ZKB_OK;
}
// Host-only: replay a scripted sequence of transcript operations through the session's own transcript code (no device work).
// ops[i]: 0 = common_scalar, 1 = write_scalar, 2 = write_point, 3 = squeeze_challenge; operands are consumed in order (scalar:
// 4 limbs, point: 8 limbs, Montgomery form); challenges are appended to `challenges` (4 limbs each).  Lets the CPU suite pin the
// framing of every transcript kind against the oracle's transcripts.
extern "C" int32_t zkb_transcript_script_host(int32_t kind, const uint8_t *ops, uint64_t n_ops, const uint64_t *operands, uint8_t *proof, uint64_t cap,
                                              uint64_t *proof_len, uint64_t *challenges) {
    ZKB_ARG(kind >= Transcript::BLAKE2B && kind <= Transcript::EVM && (ops || n_ops == 0) && proof_len);
    Transcript tr((Transcript::Kind)kind);
    const uint64_t *op = operands;
    for (uint64_t i = 0; i < n_ops; ++i) {
        switch (ops[i]) {
            case 0:
            case 1: {
                ZKB_ARG(op);
                Fr v;
                memcpy(v.l, op, 32);
                op += 4;
                if (ops[i] == 0) tr.common_scalar(v); else tr.write_scalar(v);
                break;
            }
            case 2: {
                ZKB_ARG(op);
                G1Affine p;
                memcpy(&p, op, 64);
                op += 8;
                ZKB_TRY(tr.write_point(p));
                break;
            }
            case 3: {
                ZKB_ARG(challenges);
                const Fr c = tr.squeeze();
                memcpy(challenges, c.l, 32);
                challenges += 4;
                break;
            }
            default: ZKB_ARG(false);
        }
    }
    const std::vector<uint8_t> &bytes = tr.proof();
    *proof_len = bytes.size();
    if (proof) {
        ZKB_ARG(cap >= bytes.size());
        if (!bytes.empty()) memcpy(proof, bytes.data(), bytes.size());
    }
    return ZKB_OK;
}
extern "C" int32_t zkb_keccak256_host(const uint8_t *bytes, uint64_t len, uint8_t out[32]) {
    ZKB_ARG(out && (bytes || len == 0));
    keccak256(bytes, len, out);
    return ZKB_OK;
}
// feed raw bytes to a fresh Blake2b("Halo2-Transcript") state and squeeze one Challenge255 (prefix 0x00, 64-byte digest mod r)
extern "C" int32_t zkb_blake2b_challenge_host(const uint8_t *bytes, uint64_t len, uint64_t out[4]) {
    ZKB_ARG(out && (bytes || len == 0));
    Blake2b st("Halo2-Transcript");
    if (len) st.update(bytes, len);
    const Fr c = blake2b_challenge255(st);
    memcpy(out, c.l, 32);
    return ZKB_OK;
}
