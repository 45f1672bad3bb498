//! Bodies of `ProvingKey::<G1Affine>::write` / `read` (halo2_proofs plonk.rs, PSE line) for snark-verifier-sdk's
//! `gen_pk(params, circuit, Some(path))`: the body of the file streams through the device (zkb_pk_write / zkb_pk_read) over
//! `zkb_io_vtable` callbacks around the caller's `W: Write` / `R: Read`; nothing seeks and no whole file is held.
//! The vk section is written by zkb_pk_vk_write; on reading, the fork's `VerifyingKey::read` consumes it first (as upstream does) and
//! this body checks k and num_fixed against the circuit's constraint system.  Selector bytes: the CSF carries no selectors, so a halo2
//! whose vk carries packed selectors writes / reads them itself between the vk and the body.
use crate::gpu::{check, csf, gpu};
use crate::plonk::{ConstraintSystem, ProvingKey};
use crate::poly::kzg::commitment::ParamsKZG;
use crate::SerdeFormat;
use halo2curves::bn256::{Bn256, Fr, G1Affine};
use std::io::{self, Read, Write};
use std::os::raw::c_void;

fn code(format: SerdeFormat) -> i32 {
    match format {
        SerdeFormat::Processed => 0,
        SerdeFormat::RawBytes => 1,
        SerdeFormat::RawBytesUnchecked => 2,
    }
}

struct Io<'a> {
    reader: Option<&'a mut dyn Read>,
    writer: Option<&'a mut dyn Write>,
    error: Option<io::Error>,
}

unsafe extern "C" fn io_read(user: *mut c_void, buf: *mut u8, len: u64) -> i32 {
    let io = &mut *(user as *mut Io);
    let out = std::slice::from_raw_parts_mut(buf, len as usize);
    match io.reader.as_mut().map(|r| r.read_exact(out)) {
        Some(Ok(())) => 0,
        Some(Err(e)) if e.kind() == io::ErrorKind::UnexpectedEof => ZKB_IO_EOF_CODE,
        Some(Err(e)) => {
            io.error = Some(e);
            2
        }
        None => 2,
    }
}

unsafe extern "C" fn io_write(user: *mut c_void, buf: *const u8, len: u64) -> i32 {
    let io = &mut *(user as *mut Io);
    let data = std::slice::from_raw_parts(buf, len as usize);
    match io.writer.as_mut().map(|w| w.write_all(data)) {
        Some(Ok(())) => 0,
        Some(Err(e)) => {
            io.error = Some(e);
            2
        }
        None => 2,
    }
}

const ZKB_IO_EOF_CODE: i32 = crate::zkb200_sys::ZKB_IO_EOF;

fn vtable(io: &mut Io) -> crate::zkb200_sys::zkb_io_vtable {
    crate::zkb200_sys::zkb_io_vtable { user: io as *mut Io as *mut c_void, read: io_read, write: io_write }
}

fn failed(io: Io, e: crate::plonk::Error) -> io::Error {
    io.error.unwrap_or_else(|| io::Error::new(io::ErrorKind::InvalidData, format!("{e:?}")))
}

/// `ProvingKey::write(writer, format)`: the vk section, then sections 0 - 8 (include/zkb200.h) of the device-resident key.
pub fn write<W: Write>(pk: &ProvingKey<G1Affine>, params: &ParamsKZG<Bn256>, writer: &mut W, format: SerdeFormat) -> io::Result<()> {
    let mut g = gpu();
    let h = g.proving_key(pk, params).map_err(|e| io::Error::new(io::ErrorKind::Other, format!("{e:?}")))?;
    let mut io = Io { reader: None, writer: Some(writer), error: None };
    let vt = vtable(&mut io);
    let rc = check(unsafe { crate::zkb200_sys::zkb_pk_vk_write(h, code(format), &vt) })
        .and_then(|_| check(unsafe { crate::zkb200_sys::zkb_pk_write(h, code(format), &vt) }));
    rc.map_err(|e| failed(io, e))
}

/// The body of `ProvingKey::read(reader, format)` after `VerifyingKey::read` has consumed the vk section: reads sections 0 - 8 into a
/// device-resident key for `cs` (check = true compares every derived element with the form the key derives) and returns its handle,
/// which the fork registers in the context's key cache under the vk's transcript_repr, so create_proof never rebuilds it.
pub fn read_body<R: Read>(cs: &ConstraintSystem<Fr>, params: &ParamsKZG<Bn256>, reader: &mut R, format: SerdeFormat, check_derived: bool)
    -> io::Result<*mut crate::zkb200_sys::zkb_pk> {
    let mut g = gpu();
    let srs = g.srs(params).map_err(|e| io::Error::new(io::ErrorKind::Other, format!("{e:?}")))?;
    let blob = csf::encode(cs, params.k());
    let mut io = Io { reader: Some(reader), writer: None, error: None };
    let vt = vtable(&mut io);
    let mut rep = crate::zkb200_sys::zkb_pk_read_report::default();
    let mut h = std::ptr::null_mut();
    let rc = check(unsafe {
        crate::zkb200_sys::zkb_pk_read(g.ctx, blob.as_ptr(), blob.len() as u64, code(format), &vt, srs, check_derived as i32, &mut rep, &mut h)
    });
    match rc {
        Ok(()) => Ok(h),
        Err(e) if rep.count != 0 => Err(io::Error::new(
            io::ErrorKind::InvalidData,
            format!("pk file: section {} column {}: {} bad element(s), first at {} (reason {}): {e:?}", rep.section, rep.column, rep.count,
                    rep.first_index, rep.reason),
        )),
        Err(e) => Err(failed(io, e)),
    }
}
