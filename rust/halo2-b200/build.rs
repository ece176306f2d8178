// Links libh2b200.so (built by `python -c "import __graft_entry__ as g; g.build()"` in this repository).
// H2B200_LIB_DIR = .../halo2-lib_b200 (the directory that holds libh2b200.so).
fn main() {
    let dir = std::env::var("H2B200_LIB_DIR").expect("set H2B200_LIB_DIR to the directory that holds libh2b200.so");
    println!("cargo:rustc-link-search=native={dir}");
    println!("cargo:rustc-link-lib=dylib=h2b200");
    println!("cargo:rustc-link-arg=-Wl,-rpath,{dir}");
    println!("cargo:rerun-if-env-changed=H2B200_LIB_DIR");
}
