"""The reference project's prebuilt Go CLI (go-snark-cli, built by its build-cli.sh), staged as oracle/_ref/go-snark-cli
so that tests can have the reference's own Go code verify our proofs and proving-key files.  Checker infrastructure only:
oracle/_ref/ is not under version control, and nothing of the reference is copied into the repository.

The reference checkout is GOSNARK_REFERENCE when that is set, else the first of DEFAULT_LOCATIONS that holds the binary.
Where no reference checkout exists nothing is staged, and the tests that run the binary skip or leave out that check."""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGED = os.path.join(ROOT, "oracle", "_ref", "go-snark-cli")
# a checkout named `reference` beside this repository, or at /root/reference (where the build image keeps it)
DEFAULT_LOCATIONS = (os.path.join(os.path.dirname(ROOT), "reference"), "/root/reference")


def reference_dir():
    """The reference checkout: GOSNARK_REFERENCE if set, else the first default location holding go-snark-cli; or None."""
    env = os.environ.get("GOSNARK_REFERENCE")
    for d in ((env,) if env else DEFAULT_LOCATIONS):
        if os.path.isfile(os.path.join(d, "go-snark-cli")):
            return d
    return None


def stage():
    """Copy the reference's binary to oracle/_ref/ when a reference checkout is available; the staged path or None."""
    d = reference_dir()
    src = os.path.join(d, "go-snark-cli") if d else None
    if src and (not os.path.exists(STAGED) or os.path.getsize(STAGED) != os.path.getsize(src)):
        os.makedirs(os.path.dirname(STAGED), exist_ok=True)
        shutil.copy(src, STAGED)
        os.chmod(STAGED, 0o755)
    return STAGED if os.path.exists(STAGED) else None


def require_reference_dir():
    """reference_dir() for the golden generators, which cannot run without the reference: exits with a usage message."""
    d = reference_dir()
    if not d:
        raise SystemExit("no reference checkout found: set GOSNARK_REFERENCE to a checkout of arnaucube/go-snark-study "
                         "(with its prebuilt go-snark-cli)")
    return d
