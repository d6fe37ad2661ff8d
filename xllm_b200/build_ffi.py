"""Builds the TVM-FFI drop-in modules and lays them out like FlashInfer's AOT output so that xLLM's
get_module(uri) (xllm/core/kernels/cuda/utils.cpp:371-374,526-564) loads them unchanged:

    $FLASHINFER_OPS_PATH/<uri>/<uri>.so      exporting __tvm_ffi_plan / __tvm_ffi_run | __tvm_ffi_{ragged,paged}_run

One decode module, one prefill module and the FA3 form of the prefill module (the "_sm90" URIs the reference requests for
ragged prefill on an sm90a device) are compiled (g++, apache-tvm-ffi headers) against libxllm_b200_ops.so and installed
under every URI the reference can request for bf16 (utils.cpp:388-450), by symlink.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "ffi", "tvm_ffi_modules.cc")
LIBDIR = os.path.join(HERE, "lib")
OPS_DIR = os.path.join(LIBDIR, "flashinfer_ops")


def uris():
    dec, pre = [], []
    for hd in (64, 128):
        dec.append(f"batch_decode_with_kv_cache_dtype_q_bf16_dtype_kv_bf16_dtype_o_bf16_dtype_idx_i32_head_dim_qk_{hd}_"
                   f"head_dim_vo_{hd}_posenc_0_use_swa_False_use_logits_cap_False")
        pre.append(f"batch_prefill_with_kv_cache_dtype_q_bf16_dtype_kv_bf16_dtype_o_bf16_dtype_idx_i32_head_dim_qk_{hd}_"
                   f"head_dim_vo_{hd}_posenc_0_use_swa_False_use_logits_cap_False_f16qk_False")
    return dec, pre


def uris_sm90():
    """the ragged-prefill URIs the reference requests on an sm90a device (backend "fa3": utils.cpp:376-386,417)"""
    return [u + "_sm90" for u in uris()[1]]


def build(verbose=False):
    import tvm_ffi
    root = os.path.dirname(tvm_ffi.__file__)
    inc = [os.path.join(root, "include"), "/usr/local/cuda/include"]
    dl = os.path.join(root, "include", "dlpack")           # some wheels vendor dlpack separately
    if not os.path.exists(os.path.join(inc[0], "dlpack")):
        for cand in (os.path.join(root, "3rdparty", "dlpack", "include"), dl):
            if os.path.exists(cand):
                inc.append(cand)
    os.makedirs(OPS_DIR, exist_ok=True)
    outs = {}
    for name, macro in (("xllm_b200_ffi_decode", ["-DXB_FFI_DECODE_MODULE"]), ("xllm_b200_ffi_prefill", []),
                        ("xllm_b200_ffi_prefill_sm90", ["-DXB_FFI_PREFILL_SM90_MODULE"])):
        out = os.path.join(LIBDIR, name + ".so")
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", SRC, "-o", out] + macro + [f"-I{i}" for i in inc] + [
            f"-L{LIBDIR}", "-lxllm_b200_ops", f"-L{os.path.join(root, 'lib')}", "-ltvm_ffi", "-L/usr/local/cuda/lib64", "-lcudart",
            f"-Wl,-rpath,{LIBDIR}", f"-Wl,-rpath,{os.path.join(root, 'lib')}"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("FFI module build failed")
        outs[name] = out
    dec, pre = uris()
    for lst, so in ((dec, outs["xllm_b200_ffi_decode"]), (pre, outs["xllm_b200_ffi_prefill"]),
                    (uris_sm90(), outs["xllm_b200_ffi_prefill_sm90"])):
        for uri in lst:
            d = os.path.join(OPS_DIR, uri)
            os.makedirs(d, exist_ok=True)
            link = os.path.join(d, uri + ".so")
            if os.path.lexists(link):
                os.remove(link)
            os.symlink(os.path.relpath(so, d), link)
    return OPS_DIR


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
