#!/usr/bin/env python3
"""TEST INFRASTRUCTURE: INTEGRATION.md section B made executable.

Takes the UNMODIFIED reference sources where they lie (/root/reference/src), applies -- in a temporary
directory that is deleted afterwards -- exactly the binding INTEGRATION.md shows a maintainer of the
reference (the reference's own hook.c / client.c keep everything else: interposition, the gate, the
protocol, the threads), compiles it with the reference's flags and links it against our C-ABI library:

    oracle/_ref/libnvshare_bound.so  =  reference hook + reference client  +  libnvs_engine.so

Nothing of the reference is copied into the repository: the edits below name short anchor strings of the
reference's code (file:line in the comments) and the only output is the shared object in oracle/_ref/.
tests/test_bound_reference.py runs two oversubscribed clients under the REFERENCE daemon with it.

    python oracle/bind_reference.py [--optional] [reference root] [output .so]
--optional adds the one-line optional calls of that section (copies that need no lock, recency hint, hand-over
announcement, the cap that follows what the GPU has lent) -> oracle/_ref/libnvshare_bound_opt.so
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
REF = Path(os.environ.get("REF", "/root/reference"))      # where oracle/Makefile looks too
OUT = ROOT / "oracle" / "_ref" / "libnvshare_bound.so"
BUILD = ROOT / "nvshare_b200" / "_build"

HOOK_STATE = r'''
/* ---- binding to libnvs_engine.so (INTEGRATION.md B) ---- */
#include "nvshare_engine.h"
nvs_engine *nvshare_engine;                       /* created lazily: needs the app's context; client.c uses it too */
static void *nvs_cuda_handle;
static void *nvs_resolve(const char *s) { return real_dlsym_225(nvs_cuda_handle, s); }
static nvs_engine *engine_get(void)
{
	if (!nvshare_engine) {
		nvs_engine_config cfg;
		nvs_engine_default_config(&cfg);
		cfg.resolve = nvs_resolve;                /* the REAL driver symbols, not the hooks */
		if (nvs_engine_create(&cfg, &nvshare_engine) != 0)
			log_fatal("swap engine");
	}
	return nvshare_engine;
}
'''


def edit(text, anchor, replacement, what, count=1, after=None):
    """Replace `anchor` (the first occurrence after `after`, when given) and insist that it was there."""
    start = 0
    if after is not None:
        start = text.find(after)
        assert start >= 0, f"{what}: context {after!r} not found in the reference source"
    at = text.find(anchor, start)
    assert at >= 0, f"{what}: anchor {anchor!r} not found in the reference source"
    return text[:at] + replacement + text[at + len(anchor):]


def bind_hook(src):
    # src/hook.c:50 -- file-scope state, right after the forward declaration of the real dlsym
    a = "static void *real_dlsym_225(void *handle, const char *symbol);"
    src = edit(src, a, a + HOOK_STATE, "engine state")
    # src/hook.c:145 -- remember the driver's handle for the resolver
    a = 'cuda_handle = dlopen("libcuda.so", RTLD_LAZY);'
    src = edit(src, a, a + "\n\tnvs_cuda_handle = cuda_handle;", "driver handle")
    # src/hook.c:673 -- cuMemAlloc: the allocation comes from the engine
    a = "result = real_cuMemAllocManaged(dptr, bytesize, CU_MEM_ATTACH_GLOBAL);"
    src = edit(src, a, "{ uint64_t p_ = 0; result = (CUresult)nvs_alloc(engine_get(), &p_, bytesize); "
                       "if (result == CUDA_SUCCESS) *dptr = (CUdeviceptr)p_; }", "cuMemAlloc")
    # src/hook.c:691 -- cuMemFree: ours first, the driver's for everything else
    a = "result = real_cuMemFree(dptr);"
    src = edit(src, a, "result = nvshare_engine ? (CUresult)nvs_free(nvshare_engine, dptr) : (CUresult)NVS_E_NOT_OURS;\n"
                       "\tif ((int)result == NVS_E_NOT_OURS) result = real_cuMemFree(dptr);", "cuMemFree")
    return src


def bind_client(src):
    # file scope (src/client.c:40)
    a = "pthread_t client_tid;"
    src = edit(src, a, '#include "nvshare_engine.h"\nextern nvs_engine *nvshare_engine;\n' + a, "client state")
    # src/client.c:298-304 -- LOCK_OK: fetch BEFORE the gate opens (VMM memory cannot fault)
    a = "need_lock = 0;"
    src = edit(src, a, "if (nvshare_engine) {\n\t\t\t\tif (nvs_fetch_all(nvshare_engine, NULL) != 0) log_fatal(\"fetch\");\n"
                       "\t\t\t\tnvs_set_resident_mode(nvshare_engine, 1);\n\t\t\t}\n\t\t\t" + a, "LOCK_OK", after="case LOCK_OK:")
    # src/client.c:308-317 -- DROP_LOCK: evict after the context is drained and LOCK_RELEASED is out
    a = 'log_debug("Sent %s", message_type_string[out_msg.type]);'
    src = edit(src, a, a + "\n\t\t\t\tif (nvshare_engine) {\n\t\t\t\t\tnvs_set_resident_mode(nvshare_engine, 0);\n"
                           "\t\t\t\t\tif (nvs_evict(nvshare_engine, 0, NULL) != 0) log_fatal(\"evict\");\n\t\t\t\t}",
               "DROP_LOCK", after="case DROP_LOCK:")
    # src/client.c:472-476 -- early release
    a = 'log_debug("Sent %s", message_type_string[release_msg.type]);'
    src = edit(src, a, a + "\n\t\t\tif (nvshare_engine) {\n\t\t\t\tcuda_sync_context();\n\t\t\t\tnvs_set_resident_mode(nvshare_engine, 0);\n"
                           "\t\t\t\tif (nvs_evict(nvshare_engine, 0, NULL) != 0) log_fatal(\"evict\");\n\t\t\t}", "early release")
    return src


def bind_optional(hook, client):
    """The optional calls of INTEGRATION.md B (one line each): copies that do not need the GPU, the recency hint,
    the hand-over announcement, and the cap that follows what this GPU has lent."""
    # src/hook.c:909 / :878 -- cuMemcpyHtoD / cuMemcpyDtoH on memory that is swapped out: host <-> pinned backing, no lock
    hook = edit(hook, "nvs_engine *nvshare_engine;", "nvs_engine *nvshare_engine;\nextern int own_lock;           /* src/client.c:50 */",
                "own_lock")
    a = "continue_with_lock();\n\tresult = real_cuMemcpyHtoD(dstDevice, srcHost, ByteCount);"
    hook = edit(hook, a, "if (nvshare_engine) nvs_touch(nvshare_engine, dstDevice, ByteCount);\n"
                         "\tif (!own_lock && nvshare_engine && nvs_host_io(nvshare_engine, dstDevice, (void *)srcHost, ByteCount, 1) == 0)\n"
                         "\t\treturn CUDA_SUCCESS;\n\t" + a, "HtoD bypass")
    a = "continue_with_lock();\n\tresult = real_cuMemcpyDtoH(dstHost, srcDevice, ByteCount);"
    hook = edit(hook, a, "if (!own_lock && nvshare_engine && nvs_host_io(nvshare_engine, srcDevice, dstHost, ByteCount, 0) == 0)\n"
                         "\t\treturn CUDA_SUCCESS;\n\t" + a, "DtoH bypass")
    # the same for the asynchronous flavours (src/hook.c:925, :893): for pageable-style semantics the copy may be done on return
    a = "continue_with_lock();\n\tresult = real_cuMemcpyHtoDAsync(dstDevice, srcHost, ByteCount, hStream);"
    hook = edit(hook, a, "if (nvshare_engine) nvs_touch(nvshare_engine, dstDevice, ByteCount);\n"
                         "\tif (!own_lock && nvshare_engine && nvs_host_io(nvshare_engine, dstDevice, (void *)srcHost, ByteCount, 1) == 0)\n"
                         "\t\treturn CUDA_SUCCESS;\n\t" + a, "HtoDAsync bypass")
    a = "continue_with_lock();\n\tresult = real_cuMemcpyDtoHAsync(dstHost, srcDevice, ByteCount, hStream);"
    hook = edit(hook, a, "if (!own_lock && nvshare_engine && nvs_host_io(nvshare_engine, srcDevice, dstHost, ByteCount, 0) == 0)\n"
                         "\t\treturn CUDA_SUCCESS;\n\t" + a, "DtoHAsync bypass")
    # src/hook.c:662 -- the cap follows what this GPU has lent to clients of other GPUs
    a = "if ((sum_allocated + bytesize) > nvshare_size_mem_allocatable) {"
    hook = edit(hook, a, "if ((sum_allocated + bytesize) > nvshare_size_mem_allocatable - "
                         "(nvshare_engine ? nvs_gpu_lent_bytes(nvshare_engine) : 0)) {", "cap")
    # src/client.c:313 -- DROP_LOCK, before LOCK_RELEASED is written
    a = "out_msg.type = LOCK_RELEASED;"
    client = edit(client, a, "if (nvshare_engine) nvs_evict_announce(nvshare_engine);\n\t\t\t\t" + a, "announce", after="case DROP_LOCK:")
    return hook, client


def main():
    optional = "--optional" in sys.argv
    if optional:
        sys.argv.remove("--optional")
    global REF, OUT
    REF = Path(sys.argv[1]) if len(sys.argv) > 1 else REF
    OUT = Path(sys.argv[2]) if len(sys.argv) > 2 else (OUT.with_name("libnvshare_bound_opt.so") if optional else OUT)
    src = REF / "src"
    if not os.access(src / "hook.c", os.R_OK):
        print(f"reference sources not present ({src}): nothing to bind")
        return 0
    if not (BUILD / "libnvs_engine.so").exists():
        print(f"{BUILD}/libnvs_engine.so is missing: build the product first", file=sys.stderr)
        return 1
    tmp = Path(tempfile.mkdtemp(prefix="nvs_bind_"))
    try:
        hook, client = bind_hook((src / "hook.c").read_text()), bind_client((src / "client.c").read_text())
        if optional:
            hook, client = bind_optional(hook, client)
        (tmp / "hook.c").write_text(hook)
        (tmp / "client.c").write_text(client)
        OUT.parent.mkdir(parents=True, exist_ok=True)
        cmd = ["gcc", "-O2", "-g", "-fPIC", "-w", "-D_GNU_SOURCE", f"-I{src}", f"-I{ROOT / 'include'}",
               str(tmp / "hook.c"), str(tmp / "client.c"), str(src / "common.c"), str(src / "comm.c"),
               "-shared", "-Wl,-soname=libnvshare.so", f"-Wl,--version-script={src / 'libnvshare-symbols.ld'}",
               "-Wl,--exclude-libs,ALL", f"-L{BUILD}", "-lnvs_engine", "-Wl,-rpath,$ORIGIN/../../nvshare_b200/_build",
               "-o", str(OUT), "-ldl", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            print(r.stdout + r.stderr, file=sys.stderr)
            return r.returncode
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(f"bound reference library: {OUT}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
