// Locates libllmlb_b200.so (built by `python -m llmlb_b200.build`, nvcc sm_90a) and tells rustc to
// link it.  LLMLB_B200_LIB_DIR overrides the default (../../llmlb_b200 relative to this crate).
use std::env;
use std::path::PathBuf;

fn main() {
    let dir = env::var("LLMLB_B200_LIB_DIR").map(PathBuf::from).unwrap_or_else(|_| {
        PathBuf::from(env::var("CARGO_MANIFEST_DIR").unwrap()).join("../../llmlb_b200")
    });
    println!("cargo:rustc-link-search=native={}", dir.display());
    println!("cargo:rustc-link-lib=dylib=llmlb_b200");
    println!("cargo:rustc-link-arg=-Wl,-rpath,{}", dir.display());
    println!("cargo:rerun-if-env-changed=LLMLB_B200_LIB_DIR");
    println!("cargo:rerun-if-changed=../../include/llmlb_b200.h");
}
