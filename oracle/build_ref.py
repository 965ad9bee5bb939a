"""TEST / BASELINE INFRASTRUCTURE - recipe that stages the reference's OWN hot-path source files under oracle/_ref/.

    python -m oracle.build_ref            (run by __graft_entry__.build() wherever the reference tree exists)

oracle/_ref/ is git-ignored (reference sources never enter this repository's history); a tree built where the reference
exists keeps it, so it also serves where the reference tree is absent.  There `bench.py --impl reference` / `cpu_baseline` execute
these files, UNMODIFIED, through oracle/ref_loader.py (MMF_REFERENCE_ROOT=oracle/_ref) - the reference's own
`VisualBERTBase` (BertVisioLinguisticEmbeddings + BertEncoderJit), i.e. `cpu_baseline.kind = "reference"`.
Nothing in the product (mmf_b200/) imports from here.
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.environ.get("MMF_REFERENCE_SRC", "/root/reference")
DST = os.path.join(HERE, "_ref")

# the files the fusion path executes (SURVEY.md 8a/8c); everything else they import is stubbed by ref_loader
FILES = [
    "mmf/modules/hf_layers.py",
    "mmf/modules/embeddings.py",
    "mmf/modules/vit.py",
    "mmf/models/visual_bert.py",
    "mmf/models/vilbert.py",
    "mmf/models/mmbt.py",
    "mmf/models/uniter.py",
    "mmf/models/vinvl.py",
    "mmf/models/transformers/backends/huggingface.py",
    "mmf/utils/transform.py",
    "mmf/utils/torchscript.py",
    "mmf/utils/modeling.py",
    "LICENSE",
]


def build(verbose=False):
    if not os.path.isdir(os.path.join(SRC, "mmf")):
        if os.path.isdir(os.path.join(DST, "mmf")):
            return DST                      # GPU box: use what travelled with the snapshot
        return None
    manifest = {}
    for rel in FILES:
        src = os.path.join(SRC, rel)
        if not os.path.exists(src):
            continue
        dst = os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
        with open(src, "rb") as fh:
            manifest[rel] = hashlib.sha256(fh.read()).hexdigest()
    with open(os.path.join(DST, "MANIFEST.json"), "w") as fh:
        json.dump({"source": SRC, "files": manifest}, fh, indent=1)
    if verbose:
        print("staged %d reference files under %s" % (len(manifest), DST))
    return DST


def available():
    return os.path.isdir(os.path.join(DST, "mmf", "modules"))


if __name__ == "__main__":
    print(build(verbose=True))
    sys.exit(0)
