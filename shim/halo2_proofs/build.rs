// build.rs of the fork-shaped halo2_proofs: link the H100 backend.  Not compiled in this repository's image (no cargo).
fn main() {
    let dir = std::env::var("ZKB200_LIB_DIR").expect("set ZKB200_LIB_DIR to the directory holding libzkb200.so");
    println!("cargo:rustc-link-search=native={dir}");
    println!("cargo:rustc-link-lib=dylib=zkb200");
    println!("cargo:rerun-if-env-changed=ZKB200_LIB_DIR");
}
