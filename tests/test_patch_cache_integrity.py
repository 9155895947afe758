"""The on-disk cache of compiled patch kernels (patch_fuse.cu) and the library's dynamic shared-memory limits, checked without a device.

* A cached cubin that is not a whole ELF64 image (a full disk, a writer that died) is a miss: the program is compiled again and the
  file rewritten, never handed to the loader.
* Threads of one process that compile the same program at once each write their own temporary file and rename it into place: the
  cache ends up with one whole file and no temporaries, and nobody reading the final name meanwhile sees a part of a file.
* The dynamic shared-memory limit of a kernel is shared by every handle and host thread. Every launch site raises it through one
  helper that never lowers it; a site that sets the limit itself and then launches can have it lowered by another thread in
  between. The scan below is the deterministic guard against such a site."""
import os
import re
import threading
from pathlib import Path

from maximilian_b200 import capi
from maximilian_b200.patchdef import PatchDef, R

CSRC = Path(__file__).resolve().parents[1] / "maximilian_b200" / "csrc"
ELF_HEADER = 64          # sizeof(Elf64_Ehdr)


def _new_program(salt):
    """a stage list no earlier run compiled: one of its constants comes from the process id"""
    d = PatchDef()
    d.stage("osc", d.P("f"), kind="saw", dst=R(0))
    d.stage("filter", R(0), d.K(2345.25 + (os.getpid() % 997) + salt / 64), d.K(1.5), kind="lores", dst=R(1))
    d.stage("out", R(1))
    return d


def _compile_into(directory, d, monkeypatch):
    monkeypatch.setenv("MXB_PATCH_CACHE", str(directory))
    capi.patch_codegen(d, compile=True)
    files = sorted(directory.glob("patch_*.cubin"))
    assert len(files) == 1, files
    return files[0]


def test_a_truncated_cubin_is_compiled_again_and_rewritten(tmp_path, monkeypatch):
    d = _new_program(0)
    f = _compile_into(tmp_path / "cache", d, monkeypatch)
    whole = f.read_bytes()
    assert whole[:4] == b"\x7fELF" and len(whole) > 2 * ELF_HEADER
    for cut in (len(whole) // 2, ELF_HEADER + 1, ELF_HEADER):
        f.write_bytes(whole[:cut])
        capi.patch_codegen(d, compile=True)
        assert f.read_bytes() == whole, f"a cubin cut to {cut} of {len(whole)} bytes was not rewritten"
    assert sorted(p.name for p in f.parent.iterdir()) == [f.name]


def test_threads_compiling_one_program_leave_one_whole_file(tmp_path, monkeypatch):
    """8 threads compile the same new program into one empty directory at once; a ninth reads the final name all the while"""
    d = _new_program(1)
    one = _compile_into(tmp_path / "one", d, monkeypatch).read_bytes()
    # NVRTC's output is byte-stable for one source and one set of flags, so the files below can be compared byte for byte
    assert _compile_into(tmp_path / "again", d, monkeypatch).read_bytes() == one

    shared = tmp_path / "eight"
    monkeypatch.setenv("MXB_PATCH_CACHE", str(shared))
    T = 8
    go, done = threading.Barrier(T + 1), threading.Event()
    errors, seen = [], []

    def writer():
        go.wait()
        try:
            capi.patch_codegen(d, compile=True)
        except Exception as e:          # noqa: BLE001 -- reported below, with the thread's own error text
            errors.append(e)

    def reader():
        go.wait()
        while not done.is_set():
            for p in shared.glob("patch_*.cubin") if shared.exists() else ():
                try:
                    b = p.read_bytes()
                except FileNotFoundError:
                    continue
                if b != one:
                    seen.append(len(b))

    threads = [threading.Thread(target=writer) for _ in range(T)]
    rd = threading.Thread(target=reader)
    for t in threads + [rd]:
        t.start()
    for t in threads:
        t.join()
    done.set()
    rd.join()
    assert not errors, errors
    assert not seen, f"a reader saw the cache file at {sorted(set(seen))} bytes instead of {len(one)}"
    names = sorted(p.name for p in shared.iterdir())
    assert len(names) == 1 and names[0].startswith("patch_") and names[0].endswith(".cubin"), names
    assert (shared / names[0]).read_bytes() == one


def _helper_span(text):
    """[start, end) of the definition of smem_limit_at_least in ctx.cu"""
    m = re.search(r"^int smem_limit_at_least\([^)]*\)\s*\{", text, re.M)
    assert m, "ctx.cu defines no smem_limit_at_least"
    end = text.index("\n}\n", m.end())
    return m.start(), end


def test_every_shared_memory_limit_goes_through_the_one_helper():
    pattern = re.compile(r"MaxDynamicSharedMemorySize|MAX_DYNAMIC_SHARED_SIZE_BYTES|FuncSetAttribute|KernelSetAttribute")
    ctx = (CSRC / "ctx.cu").read_text()
    lo, hi = _helper_span(ctx)
    inside, outside = 0, []
    for p in sorted(CSRC.rglob("*")):
        if not p.is_file():
            continue
        text = p.read_text(errors="replace")
        for m in pattern.finditer(text):
            if p.name == "ctx.cu" and lo <= m.start() < hi:
                inside += 1
            else:
                outside.append(f"{p.relative_to(CSRC)}:{text.count(chr(10), 0, m.start()) + 1}: {m.group(0)}")
    assert not outside, "a kernel's dynamic shared-memory limit is set outside smem_limit_at_least:\n" + "\n".join(outside)
    assert inside >= 1, "smem_limit_at_least no longer sets the limit"
    # and every launch site that used to set it calls the helper instead
    calls = {p.name: len(re.findall(r"\bsmem_limit_at_least\(", p.read_text())) for p in CSRC.glob("*.cu*")}
    assert calls["patch.cu"] >= 1 and calls["delay_impl.cuh"] >= 1 and calls["spectral.cu"] >= 5, calls
