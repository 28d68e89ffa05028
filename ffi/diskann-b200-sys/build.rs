// Locates libdiskann_b200.so (built by `make -C diskann_b200/csrc`, nvcc sm_90a) — the library is not
// compiled by cargo: it needs nvcc, and the workspace must stay buildable on machines without CUDA.
use std::env;
use std::path::PathBuf;

fn main() {
    println!("cargo:rerun-if-env-changed=DISKANN_B200_LIB_DIR");
    let dir = env::var("DISKANN_B200_LIB_DIR").map(PathBuf::from).unwrap_or_else(|_| {
        // default: the repository layout (ffi/diskann-b200-sys -> ../../diskann_b200)
        PathBuf::from(env::var("CARGO_MANIFEST_DIR").unwrap()).join("../../diskann_b200")
    });
    println!("cargo:rustc-link-search=native={}", dir.display());
    println!("cargo:rustc-link-lib=dylib=diskann_b200");
    println!("cargo:rustc-link-arg=-Wl,-rpath,{}", dir.display());
}
