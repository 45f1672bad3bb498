//! Bodies of `ParamsKZG::<Bn256>::read_custom` / `write_custom` (halo2_proofs 1.1.0 src/poly/kzg/commitment.rs) for the file the
//! reference loads with `load_params` (prover/src/utils.rs:39-83).  The 2 * 2^k G1 points are decoded or encoded on the GPU
//! (zkb_g1_decode / zkb_g1_encode, streamed through pinned buffers); the two G2 points on the host (zkb_g2_*_host).
//! Bodies of `ParamsKZG::<Bn256>::setup` / `unsafe_setup_with_s` / `new`: g and g_lagrange generated on the GPU (zkb_srs_setup_dev),
//! g2 and s_g2 on the host (zkb_g2_setup_host).  The random s of `setup` / `new` is drawn here in Rust; no RNG crosses the C ABI.
use crate::gpu::{check, gpu};
use crate::poly::kzg::commitment::ParamsKZG;
use crate::zkb200_sys::*;
use crate::SerdeFormat;
use ff::Field;
use halo2curves::bn256::{Bn256, Fr, G1Affine, G2Affine};
use rand_core::{OsRng, RngCore};
use std::io::{self, Read, Write};
use std::os::raw::c_void;

/// `ParamsKZG::unsafe_setup_with_s(k, s)`: g[i] = [s^i] G1, g_lagrange[i] = [L_i(s)] G1, g2, s_g2 = [s] g2.  When s^n = 1 the
/// Lagrange basis is returned where upstream's `invert().unwrap()` panics (include/zkb200.h).
pub fn unsafe_setup_with_s(k: u32, s: Fr) -> ParamsKZG<Bn256> {
    let n = 1usize << k;
    let bytes = (n * std::mem::size_of::<G1Affine>()) as u64;
    let s_raw = &s as *const Fr as *const u64;
    let mut g_host = vec![G1Affine::default(); n];
    let mut gl_host = vec![G1Affine::default(); n];
    {
        let g = gpu();
        let (mut d_g, mut d_gl): (*mut c_void, *mut c_void) = (std::ptr::null_mut(), std::ptr::null_mut());
        check(unsafe { zkb_malloc(g.ctx, bytes, &mut d_g) }).expect("zkb_malloc g");
        check(unsafe { zkb_malloc(g.ctx, bytes, &mut d_gl) }).expect("zkb_malloc g_lagrange");
        check(unsafe { zkb_srs_setup_dev(g.ctx, k, s_raw, d_g as *mut u64, d_gl as *mut u64, std::ptr::null_mut()) }).expect("zkb_srs_setup_dev");
        check(unsafe { zkb_d2h(g.ctx, g_host.as_mut_ptr() as *mut c_void, d_g, bytes) }).expect("zkb_d2h g");
        check(unsafe { zkb_d2h(g.ctx, gl_host.as_mut_ptr() as *mut c_void, d_gl, bytes) }).expect("zkb_d2h g_lagrange");
        check(unsafe { zkb_free(g.ctx, d_g) }).expect("zkb_free");
        check(unsafe { zkb_free(g.ctx, d_gl) }).expect("zkb_free");
    }
    let (mut g2, mut s_g2) = (G2Affine::default(), G2Affine::default());
    check(unsafe { zkb_g2_setup_host(s_raw, &mut g2 as *mut G2Affine as *mut u64, &mut s_g2 as *mut G2Affine as *mut u64) })
        .expect("zkb_g2_setup_host");
    ParamsKZG::from_parts(k, n as u64, g_host, gl_host, g2, s_g2)
}

/// `ParamsKZG::setup(k, rng)`: s = Fr::random(rng), then `unsafe_setup_with_s`.
pub fn setup<R: RngCore>(k: u32, rng: R) -> ParamsKZG<Bn256> {
    unsafe_setup_with_s(k, Fr::random(rng))
}

/// `ParamsKZG::new(k)`: `setup` with the operating system's RNG.
pub fn new(k: u32) -> ParamsKZG<Bn256> {
    setup(k, OsRng)
}

fn code(format: SerdeFormat) -> i32 {
    match format {
        SerdeFormat::Processed => 0,
        SerdeFormat::RawBytes => 1,
        SerdeFormat::RawBytesUnchecked => 2,
    }
}

fn g1_len(format: SerdeFormat) -> usize {
    if let SerdeFormat::Processed = format { 32 } else { 64 }
}

fn invalid(msg: String) -> io::Error {
    io::Error::new(io::ErrorKind::InvalidData, msg)
}

fn read_g1<R: Read>(reader: &mut R, name: &str, n: usize, format: SerdeFormat) -> io::Result<Vec<G1Affine>> {
    let mut bytes = vec![0u8; n * g1_len(format)];
    reader.read_exact(&mut bytes)?;
    let mut out = vec![G1Affine::default(); n];
    let mut rep = zkb_decode_report::default();
    let g = gpu();
    check(unsafe { zkb_g1_decode(g.ctx, code(format), bytes.as_ptr(), n as u64, out.as_mut_ptr() as *mut u64, &mut rep, std::ptr::null_mut()) })
        .map_err(|e| invalid(format!("{name}: {e:?}")))?;
    if rep.count != 0 {
        return Err(invalid(format!("{name}[{}]: bad point (reason {}); {} bad point(s) in {name}", rep.first_bad, rep.reason, rep.count)));
    }
    Ok(out)
}

fn read_g2<R: Read>(reader: &mut R, name: &str, format: SerdeFormat) -> io::Result<G2Affine> {
    let mut bytes = vec![0u8; 2 * g1_len(format)];
    reader.read_exact(&mut bytes)?;
    let mut out = G2Affine::default();
    let mut status = 0i32;
    check(unsafe { zkb_g2_decode_host(code(format), bytes.as_ptr(), &mut out as *mut G2Affine as *mut u64, &mut status) })
        .map_err(|e| invalid(format!("{name}: {e:?}")))?;
    if status != 0 {
        return Err(invalid(format!("{name}: bad point (reason {status})")));
    }
    Ok(out)
}

pub fn read_custom<R: Read>(reader: &mut R, format: SerdeFormat) -> io::Result<ParamsKZG<Bn256>> {
    let mut k = [0u8; 4];
    reader.read_exact(&mut k)?;
    let k = u32::from_le_bytes(k);
    let n = 1usize << k;
    let g = read_g1(reader, "g", n, format)?;
    let g_lagrange = read_g1(reader, "g_lagrange", n, format)?;
    let g2 = read_g2(reader, "g2", format)?;
    let s_g2 = read_g2(reader, "s_g2", format)?;
    Ok(ParamsKZG::from_parts(k, n as u64, g, g_lagrange, g2, s_g2))
}

fn write_g1<W: Write>(writer: &mut W, points: &[G1Affine], format: SerdeFormat) -> io::Result<()> {
    let mut bytes = vec![0u8; points.len() * g1_len(format)];
    let g = gpu();
    check(unsafe { zkb_g1_encode(g.ctx, code(format), points.as_ptr() as *const u64, points.len() as u64, bytes.as_mut_ptr(), std::ptr::null_mut()) })
        .map_err(|e| invalid(format!("{e:?}")))?;
    writer.write_all(&bytes)
}

fn write_g2<W: Write>(writer: &mut W, p: &G2Affine, format: SerdeFormat) -> io::Result<()> {
    let mut bytes = vec![0u8; 2 * g1_len(format)];
    check(unsafe { zkb_g2_encode_host(code(format), p as *const G2Affine as *const u64, bytes.as_mut_ptr()) }).map_err(|e| invalid(format!("{e:?}")))?;
    writer.write_all(&bytes)
}

pub fn write_custom<W: Write>(params: &ParamsKZG<Bn256>, writer: &mut W, format: SerdeFormat) -> io::Result<()> {
    writer.write_all(&params.k().to_le_bytes())?;
    write_g1(writer, params.get_g(), format)?;
    write_g1(writer, params.g_lagrange(), format)?;
    write_g2(writer, &params.g2(), format)?;
    write_g2(writer, &params.s_g2(), format)
}
