//! `plonk::create_proof` on the H100 proving session.  Same signature, same transcript traffic, same RNG draws as the CPU crate
//! (halo2_proofs 1.1.0 @ e5ddf67 src/plonk/prover.rs); called unchanged from circuit-benchmarks/src/super_circuit.rs:117-132,
//! circuit-benchmarks/src/packed_multi_keccak.rs:72-87 and, through snark-verifier-sdk, prover/src/common/prover/utils.rs:31.
//!
//! What stays in Rust: `Circuit::synthesize` per phase (WitnessCollection, batch_invert_assigned), the blinding rows and every other
//! RNG draw, the transcript object `T`.  What moves to the device: everything between two transcript operations -- commitments
//! (MSM), basis changes (NTT), mv-lookup multiplicities and grand sums, permutation grand products, the quotient, evaluations, SHPLONK.
use super::{Circuit, Error, ProvingKey};
use crate::gpu::{self, check, transcript::Bridge};
use crate::poly::kzg::commitment::{KZGCommitmentScheme, ParamsKZG};
use crate::poly::kzg::multiopen::ProverSHPLONK;
use crate::transcript::{EncodedChallenge, TranscriptWrite};
use crate::zkb200_sys::*;
use ff::Field;
use halo2curves::bn256::{Bn256, Fr, G1Affine};
use rand_core::RngCore;

pub fn create_proof<'params, E, R, T, ConcreteCircuit>(
    params: &'params ParamsKZG<Bn256>,
    pk: &ProvingKey<G1Affine>,
    circuits: &[ConcreteCircuit],
    instances: &[&[&[Fr]]],
    mut rng: R,
    transcript: &mut T,
) -> Result<(), Error>
where
    E: EncodedChallenge<G1Affine>,
    R: RngCore,
    T: TranscriptWrite<G1Affine, E>,
    ConcreteCircuit: Circuit<Fr>,
{
    // the session proves ONE circuit per call; halo2 interleaves several circuits per proof only in tests the reference does not run
    assert_eq!(circuits.len(), 1, "libzkb200 proves one circuit instance per create_proof call");
    let cs = pk.get_vk().cs();
    let n = 1usize << params.k();
    let bf = cs.blinding_factors();
    let unusable = bf + 1;

    let mut g = gpu::gpu();
    let gpk = g.proving_key(pk, params)?;
    let mut bridge = Bridge::<E, T>::new(transcript);
    let vt = bridge.vtable();

    // vk.hash_into(transcript) and the instance scalars are absorbed by the session through the callbacks (KZG: QUERY_INSTANCE = false)
    let inst_ptrs: Vec<*const u64> = instances[0].iter().map(|c| c.as_ptr() as *const u64).collect();
    let inst_lens: Vec<u32> = instances[0].iter().map(|c| c.len() as u32).collect();
    let repr: Fr = pk.get_vk().transcript_repr();
    let mut sess = std::ptr::null_mut();
    check(unsafe { zkb_prove_begin_cb(gpk, &vt, &repr as *const Fr as *const u64, inst_ptrs.as_ptr(), inst_lens.as_ptr(), &mut sess) })?;
    let guard = SessionGuard(sess);

    // ---- advice, phase by phase: unchanged Rust synthesis, then one call per phase
    let mut challenges = vec![Fr::ZERO; cs.num_challenges()];
    let mut advice: Vec<Vec<Fr>> = vec![Vec::new(); cs.num_advice_columns()];
    for phase in cs.phases() {
        let cols = super::witness::synthesize_phase(&circuits[0], cs, params.k(), phase, instances[0], &challenges, unusable)?; // WitnessCollection + batch_invert_assigned
        for (c, mut values) in cols {
            for v in values[n - unusable..].iter_mut() {
                *v = Fr::random(&mut rng); // blinding rows, same draw order as upstream (column order, row order)
            }
            advice[c] = values;
        }
        let ptrs: Vec<*const u64> = advice
            .iter()
            .enumerate()
            .map(|(c, v)| if cs.advice_column_phase()[c] == phase.to_u8() { v.as_ptr() as *const u64 } else { std::ptr::null() })
            .collect();
        let mut ch = vec![[0u64; 4]; cs.num_challenges().max(1)];
        check(unsafe { zkb_prove_advice_phase(sess, phase.to_u8() as u32, ptrs.as_ptr(), ch.as_mut_ptr() as *mut u64) })?;
        for (i, p) in cs.challenge_phase().iter().enumerate() {
            if *p == phase.to_u8() {
                challenges[i] = unsafe { std::mem::transmute_copy(&ch[i]) };
            }
        }
    }

    // ---- remaining RNG draws, in upstream order: mv-lookup phi blinds per lookup, permutation z blinds per set, vanishing random poly
    let n_sets = (cs.permutation().get_columns().len() + cs.degree() - 3) / (cs.degree() - 2);
    let phi_blinds: Vec<Fr> = (0..cs.lookups().len() * bf).map(|_| Fr::random(&mut rng)).collect();
    let z_blinds: Vec<Fr> = (0..n_sets * bf).map(|_| Fr::random(&mut rng)).collect();
    let random_poly: Vec<Fr> = (0..n).map(|_| Fr::random(&mut rng)).collect();
    // NOTE (SURVEY.md 8c): the relative order of these three groups of draws is the one fact of create_proof this repository could not
    // pin without running the Rust crate; diff one proof against the CPU crate with a fixed seed before relying on byte equality.

    let mut len = 0u64;
    check(unsafe {
        zkb_prove_finish(sess, z_blinds.as_ptr() as *const u64, phi_blinds.as_ptr() as *const u64, random_poly.as_ptr() as *const u64,
                         std::ptr::null_mut(), 0, &mut len)
    })?;
    drop(guard);
    if let Some(e) = bridge.io_error.take() {
        return Err(Error::Transcript(e));
    }
    Ok(())
}

struct SessionGuard(*mut zkb_session);
impl Drop for SessionGuard {
    fn drop(&mut self) {
        unsafe { zkb_session_destroy(self.0) };
    }
}

// type-level reminder of what this body is instantiated with on the reference's call sites
#[allow(dead_code)]
type Instantiation<'a> = (KZGCommitmentScheme<Bn256>, ProverSHPLONK<'a, Bn256>);
