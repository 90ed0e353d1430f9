"""Stage the UNMODIFIED reference files the checkers and baselines execute as ONE archive under oracle/_ref/ (git-ignored build
output, like the compiled .so: it stays out of history but travels to the GPU box with the tree because it is not in
.gpurunignore; /root/reference itself does not exist there).

    python oracle/build_ref.py            # run where /root/reference exists (the build container); __graft_entry__.build() calls it

The reference is pure Python: "building" it is copying the files where they lie.  Nothing here is edited, and nothing
under wsl4mis_b200/ or dropin/ may import from oracle/_ref (tests/test_abi_cpu.py checks).  Users of the staged files:
  * bench.py --impl reference     the reference's own modules on the host CPU (cpu_baseline kind "reference")
  * bench.py gpu_baseline         the same modules on cuda: stock PyTorch on the same GPU, the real kernel to beat
  * tests/test_gpu_scripts.py     runs the reference's train_*.py scripts UNCHANGED on top of dropin/ (SURVEY 8(b))
"""
import hashlib
import io
import json
import os
import sys
import tarfile
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/code"
OUT = os.path.join(HERE, "_ref")
TAR = os.path.join(OUT, "reference_code.tar")          # the staged artefact: one archive + a sha256 manifest

FILES = [
    "networks/unet.py", "networks/pnet.py",
    "utils/losses.py", "utils/gate_crf_loss.py", "utils/ramps.py", "utils/metrics.py",
    "dataloaders/utils.py", "val_2D.py",
    "train_weakly_supervised_pCE_2D.py", "train_weakly_supervised_pCE_GatedCRFLoss_2D.py",
    "train_weakly_supervised_pCE_MumfordShah_Loss_2D.py", "train_weakly_supervised_pCE_TV_2D.py",
    "train_weakly_supervised_pCE_Entropy_Mini_2D.py", "train_weakly_supervised_segmentation_pCE_ours_proposed.py",
    "train_weakly_supervised_ustm_2D.py", "train_uncertainty_aware_mean_teacher_2D.py",
]


def build(verbose=True):
    """-> True when a staged archive exists afterwards"""
    if not os.path.isdir(REF):
        if verbose:
            print(f"{REF} not present: keeping whatever is staged in {OUT}")
        return os.path.exists(TAR)
    os.makedirs(OUT, exist_ok=True)
    manifest = {}
    with tarfile.open(TAR, "w") as tar:
        for rel in FILES:
            data = open(os.path.join(REF, rel), "rb").read()
            manifest[rel] = hashlib.sha256(data).hexdigest()
            info = tarfile.TarInfo("code/" + rel)
            info.size = len(data)
            tar.addfile(info, io.BytesIO(data))
    json.dump(manifest, open(os.path.join(OUT, "MANIFEST.json"), "w"), indent=1)
    if verbose:
        print(f"staged {len(FILES)} unmodified reference files into {TAR}")
    return True


def extract(dst=None):
    """Unpack the staged archive into `dst` (default: a fresh temporary directory) and return <dst>/code, or None when nothing
    is staged.  The bytes are checked against the manifest written at staging time."""
    if not os.path.exists(TAR):
        return None
    dst = dst or tempfile.mkdtemp(prefix="wsl4mis_ref_")
    manifest = json.load(open(os.path.join(OUT, "MANIFEST.json")))
    with tarfile.open(TAR) as tar:
        tar.extractall(dst, filter="data")
    for rel, sha in manifest.items():
        assert hashlib.sha256(open(os.path.join(dst, "code", rel), "rb").read()).hexdigest() == sha, rel
    return os.path.join(dst, "code")


if __name__ == "__main__":
    sys.exit(0 if build() else 1)
