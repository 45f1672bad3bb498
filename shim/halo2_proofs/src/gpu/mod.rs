//! Process-global H100 context and caches.  Callers of the reference serialise proving behind a `Mutex<Prover>`
//! (prover/src/test/inner.rs:20-30) and may call from any thread, so the context is lazily created once and guarded by a mutex;
//! one proof at a time per device, exactly as the library requires.  There is NO CPU fallback: a missing device is an error.
pub mod csf;
pub mod transcript;

use crate::zkb200_sys::*;
use std::collections::HashMap;
use std::ffi::CStr;
use std::sync::{Mutex, OnceLock};

pub struct Gpu {
    pub ctx: *mut zkb_ctx,
    srs_by_k: HashMap<(u32, [u64; 8]), *mut zkb_srs>,       // keyed by (k, first SRS point): one upload per params file
    pk_by_vk: HashMap<[u8; 32], *mut zkb_pk>,               // keyed by vk.transcript_repr (like prover::pk_map, prover/src/common/prover.rs:23)
}
unsafe impl Send for Gpu {}

static GPU: OnceLock<Mutex<Gpu>> = OnceLock::new();

pub fn gpu() -> std::sync::MutexGuard<'static, Gpu> {
    GPU.get_or_init(|| {
        let device: i32 = std::env::var("ZKB200_DEVICE").ok().and_then(|v| v.parse().ok()).unwrap_or(0);
        let mut ctx = std::ptr::null_mut();
        check(unsafe { zkb_init(device, &mut ctx) }).expect("libzkb200: no usable H100 (there is no CPU fallback)");
        Mutex::new(Gpu { ctx, srs_by_k: HashMap::new(), pk_by_vk: HashMap::new() })
    })
    .lock()
    .unwrap()
}

pub fn check(rc: i32) -> Result<(), crate::plonk::Error> {
    if rc == 0 {
        return Ok(());
    }
    let msg = unsafe { CStr::from_ptr(zkb_last_error()) }.to_string_lossy().into_owned();
    log::error!("libzkb200 error {rc}: {msg}");
    // -2 (invalid argument) is what an unsatisfied lookup / malformed witness produces; everything else is a backend failure
    Err(if rc == -2 { crate::plonk::Error::Synthesis } else { crate::plonk::Error::BackendFailure(msg) })
}

impl Gpu {
    /// ParamsKZG -> device-resident handle (zkb_srs_load); `ParamsKZG::downsize` maps to zkb_srs_downsize on the cached parent
    pub fn srs(&mut self, params: &crate::poly::kzg::commitment::ParamsKZG<halo2curves::bn256::Bn256>) -> Result<*mut zkb_srs, crate::plonk::Error> {
        let g = params.get_g();
        let gl = params.g_lagrange();
        let key = (params.k(), unsafe { std::mem::transmute_copy::<_, [u64; 8]>(&g[0]) });
        if let Some(&h) = self.srs_by_k.get(&key) {
            return Ok(h);
        }
        let mut h = std::ptr::null_mut();
        check(unsafe { zkb_srs_load(self.ctx, params.k(), g.as_ptr() as *const u64, gl.as_ptr() as *const u64, &mut h) })?;
        self.srs_by_k.insert(key, h);
        Ok(h)
    }

    /// ProvingKey -> device-resident key (fixed / sigma columns, coset cache), built once per circuit
    pub fn proving_key(
        &mut self,
        pk: &crate::plonk::ProvingKey<halo2curves::bn256::G1Affine>,
        params: &crate::poly::kzg::commitment::ParamsKZG<halo2curves::bn256::Bn256>,
    ) -> Result<*mut zkb_pk, crate::plonk::Error> {
        let key: [u8; 32] = pk.get_vk().transcript_repr().to_repr();
        if let Some(&h) = self.pk_by_vk.get(&key) {
            return Ok(h);
        }
        let srs = self.srs(params)?;
        let blob = csf::encode(pk.get_vk().cs(), params.k());
        let fixed: Vec<*const u64> = pk.fixed_values.iter().map(|c| c.as_ptr() as *const u64).collect();
        let sigma: Vec<*const u64> = pk.permutation.permutations.iter().map(|c| c.as_ptr() as *const u64).collect();
        let mut h = std::ptr::null_mut();
        check(unsafe { zkb_pk_create_with_srs(self.ctx, blob.as_ptr(), blob.len() as u64, fixed.as_ptr(), sigma.as_ptr(), srs, &mut h) })?;
        self.pk_by_vk.insert(key, h);
        Ok(h)
    }
}
