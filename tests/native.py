"""TEST INFRASTRUCTURE — builds the shared libraries of the test-side native code (the host emulation in tests/emu, the
plain-C references in tests/*_ref).  Never part of the product."""
import os
import subprocess
import tempfile


def shared_library(out_dir, name, cmd, deps):
    """Path of library `name` in `out_dir`, compiled by `cmd` (the compiler's argument list; "-o <file>" is appended)
    when it is missing or older than any file in `deps`.  The compiler writes a file of this process's own next to
    the library, which then replaces it: a process that loads the library never sees it half written, however many
    processes build it at once.  A temporary directory stands in for `out_dir` when that is not writable."""
    try:
        os.makedirs(out_dir, exist_ok=True)
        if not os.access(out_dir, os.W_OK):
            raise OSError
    except OSError:
        out_dir = tempfile.mkdtemp(prefix="kao_%s_" % name.split(".")[0])
    so = os.path.join(out_dir, name)
    if os.path.exists(so) and os.path.getmtime(so) >= max(os.path.getmtime(d) for d in deps):
        return so
    tmp = "%s.%d.tmp" % (so, os.getpid())
    try:
        subprocess.check_call(list(cmd) + ["-o", tmp])
        os.replace(tmp, so)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    return so
