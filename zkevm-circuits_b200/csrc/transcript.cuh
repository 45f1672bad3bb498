// transcript.cuh -- the transcript of a proving session: what the prover absorbs, what it squeezes and the proof bytes it writes.
#pragma once
#include "common.cuh"
#include "blake2b.h"
#include "poseidon.h"

namespace zkb {

class Transcript {
public:
    enum Kind : int32_t {
        BLAKE2B = 0,    // Blake2bWrite<_, G1Affine, Challenge255<_>> (the benches)
        POSEIDON = 1,   // snark-verifier-sdk PoseidonTranscript (gen_snark_shplonk)
        EVM = 2,        // snark-verifier EvmTranscript over Keccak-256 (gen_evm_proof_shplonk)
        CALLER = 3,     // the caller's transcript through zkb_transcript_vtable: create_proof's generic `T: TranscriptWrite`, whose four
                        // operations the shim forwards to the Rust object it was handed
    };
    explicit Transcript(Kind kind = BLAKE2B, const zkb_transcript_vtable *vt = nullptr) : kind(kind) { if (vt) this->vt = *vt; }
    void common_scalar(const Fr &v);
    void write_scalar(const Fr &v);
    // fails at once for the point at infinity and when the caller's transcript refuses the point
    int32_t write_point(const G1Affine &p);
    Fr squeeze();
    // the first failure a caller's callback reported: the other operations return nothing, so their callbacks' errors surface here
    int32_t status() const;
    const std::vector<uint8_t> &proof() const { return bytes; }

private:
    Kind kind;
    zkb_transcript_vtable vt{};
    int32_t cb_error = 0;   // first non-zero return of a caller callback
    Blake2b b2{"Halo2-Transcript"};
    PoseidonSponge pos;
    std::vector<uint8_t> evm_buf;
    std::vector<uint8_t> bytes;
    void callback(int32_t r) { if (r && !cb_error) cb_error = r; }
};

}  // namespace zkb
