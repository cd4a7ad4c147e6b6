"""Builds oracle/_ref/: the reference's OWN loss / composer / correspondence-finder sources, made importable.

TEST INFRASTRUCTURE (needs a checkout of the reference, PDC_REFERENCE_ROOT).  Nothing is copied into the repository:
the reference files are read where they lie, a short list of documented, LINE-ANCHORED Python-2 -> Python-3
patches is applied in memory, and the result is written to the git-ignored directory oracle/_ref/ (it travels to
a test machine like a built .so, but never enters history).  Every patch names the reference line it
touches and must match that line's text exactly, so a different reference revision fails loudly instead of being
silently mis-patched.  What is executed afterwards IS the reference's code:

    dense_correspondence/loss_functions/pixelwise_contrastive_loss.py      (411 lines, 5 patched)
    dense_correspondence/loss_functions/loss_composer.py                   (218 lines, 6 patched)
    dense_correspondence/correspondence_tools/correspondence_finder.py     (619 lines, 4 patched)

plus three stub modules that hold ONLY text cut out of the reference (the classes / functions the files above
import from modules that cannot be imported here because they pull in the 100 GB dataset stack, cv2, yaml configs):

    dense_correspondence/dataset/spartan_dataset_masked.py      SpartanDatasetDataType (:31-36), SpartanDataset.{empty_tensor,
                                                                is_empty} (dense_correspondence_dataset_masked.py:209-223),
                                                                create_non_matches (:841-858), flatten_uv_tensor (:1255-1264)
    dense_correspondence_manipulation/utils/constants.py        DEPTH_IM_SCALE (constants.py:10) + `utils`
    dense_correspondence_manipulation/utils/utils.py            flattened_pixel_locations_to_u_v (utils.py:312-323)

    python oracle/build_ref.py            # writes oracle/_ref/, prints the patch list
"""
import os
import re
import sys
import textwrap

# a checkout of RobotLocomotion/pytorch-dense-correspondence (with its external/ submodules)
REF_ROOT = os.environ.get("PDC_REFERENCE_ROOT") or None
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")

# (line number, exact old substring, new substring, why)
PATCHES = {
    "dense_correspondence/loss_functions/pixelwise_contrastive_loss.py": [
        (8, "    \tself.type", "        self.type", "py2 tab = column 8; py3 raises TabError"),
        (113, "num_non_matches / num_matches", "num_non_matches // num_matches", "py2 int / int is floor division"),
        (295, "long(non_match_loss_vec", "int(non_match_loss_vec", "py2 long -> py3 int"),
        (321, "len(non_matches_b)/len(matches_b)", "len(non_matches_b)//len(matches_b)", "py2 int / int is floor division"),
        (351, "u_v_pixel_locations[:,1]/self.image_width", "u_v_pixel_locations[:,1]//self.image_width",
         "torch 1.1 LongTensor / int is integer division; torch >= 1.5 would produce floats"),
    ],
    "dense_correspondence/loss_functions/loss_composer.py": [
        (28, 'print "applying SINGLE_OBJECT_WITHIN_SCENE loss"', 'print("applying SINGLE_OBJECT_WITHIN_SCENE loss")', "print statement"),
        (37, 'print "applying SINGLE_OBJECT_ACROSS_SCENE loss"', 'print("applying SINGLE_OBJECT_ACROSS_SCENE loss")', "print statement"),
        (43, 'print "applying DIFFERENT_OBJECT loss"', 'print("applying DIFFERENT_OBJECT loss")', "print statement"),
        (50, 'print "applying MULTI_OBJECT loss"', 'print("applying MULTI_OBJECT loss")', "print statement"),
        (59, 'print "applying SYNTHETIC_MULTI_OBJECT loss"', 'print("applying SYNTHETIC_MULTI_OBJECT loss")', "print statement"),
        (215, "Variable(torch.FloatTensor([0]).cuda())", "Variable(torch.FloatTensor([0]))",
         "the oracle runs on the CPU; value unchanged"),
    ],
    "dense_correspondence/correspondence_tools/correspondence_finder.py": [
        (322, 'print "warning, empty mask b"', 'print("warning, empty mask b")', "print statement"),
        (329, "randomized_mask_b_indices_flat/image_width", "randomized_mask_b_indices_flat//image_width",
         "torch 1.1 LongTensor / int is integer division"),
        (346, "diffs_0.view(-1,1)", "diffs_0.contiguous().view(-1,1)",
         "torch 1.1 returned a contiguous result for (transposed - tensor); torch >= 1.5 keeps the transposed strides and .view raises"),
        (347, "diffs_1.view(-1,1)", "diffs_1.contiguous().view(-1,1)", "same"),
    ],
}

# text cut out of the reference: (file, first line, last line, expected first-line text)
CUTS = {
    "datatype": ("dense_correspondence/dataset/spartan_dataset_masked.py", 31, 36, "class SpartanDatasetDataType:"),
    "empty_is_empty": ("dense_correspondence/dataset/dense_correspondence_dataset_masked.py", 209, 223, "    @staticmethod"),
    "create_non_matches": ("dense_correspondence/dataset/spartan_dataset_masked.py", 841, 858,
                           "    def create_non_matches(self, uv_a, uv_b_non_matches, multiplier):"),
    "flatten_uv_tensor": ("dense_correspondence/dataset/spartan_dataset_masked.py", 1255, 1264, "    @staticmethod"),
    "depth_scale": ("modules/dense_correspondence_manipulation/utils/constants.py", 10, 10, "DEPTH_IM_SCALE = 1000.0"),
    "flat_to_uv": ("modules/dense_correspondence_manipulation/utils/utils.py", 312, 323,
                   "def flattened_pixel_locations_to_u_v(flat_pixel_locations, image_width):"),
}


def reference_available():
    return REF_ROOT is not None and all(os.path.isfile(os.path.join(REF_ROOT, p)) for p in PATCHES)


def _lines(rel):
    with open(os.path.join(REF_ROOT, rel), "r") as f:
        return f.read().split("\n")


def _patched(rel, log):
    lines = _lines(rel)
    for ln, old, new, why in PATCHES[rel]:
        cur = lines[ln - 1]
        if old not in cur:
            raise RuntimeError("%s:%d does not contain %r (reference revision differs?): %r" % (rel, ln, old, cur))
        lines[ln - 1] = cur.replace(old, new, 1)
        log.append("%s:%d  %s  [%s]" % (rel, ln, why, old.strip()))
    return "\n".join(lines)


def _cut(key):
    rel, a, b, first = CUTS[key]
    lines = _lines(rel)[a - 1:b]
    if not lines[0].startswith(first):
        raise RuntimeError("%s:%d expected %r, found %r" % (rel, a, first, lines[0]))
    return "\n".join(lines)


def _write(rel, text):
    path = os.path.join(OUT, rel)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write(text if text.endswith("\n") else text + "\n")


def build(verbose=False):
    if not reference_available():
        raise RuntimeError("set PDC_REFERENCE_ROOT to a checkout of the reference (now %r)" % REF_ROOT)
    log = []
    for rel in PATCHES:
        _write(rel, "# GENERATED by oracle/build_ref.py from %s/%s -- do not commit\n" % (REF_ROOT, rel) + _patched(rel, log))
    stub = ["# GENERATED by oracle/build_ref.py: text cut out of the reference, see the module docstring there", "import torch", "",
            _cut("datatype"), "", "class SpartanDataset(object):", _cut("empty_is_empty"), "", _cut("create_non_matches"), "",
            _cut("flatten_uv_tensor"), ""]
    _write("dense_correspondence/dataset/spartan_dataset_masked.py", "\n".join(stub))
    flat = _cut("flat_to_uv").replace("flat_pixel_locations/image_width", "flat_pixel_locations//image_width")
    log.append("modules/dense_correspondence_manipulation/utils/utils.py:323  torch 1.1 LongTensor / int is integer division  "
               "[flat_pixel_locations/image_width]")
    _write("dense_correspondence_manipulation/utils/utils.py", "# GENERATED by oracle/build_ref.py\n" + flat)
    _write("dense_correspondence_manipulation/utils/constants.py",
           "# GENERATED by oracle/build_ref.py\nfrom dense_correspondence_manipulation.utils import utils\n" + _cut("depth_scale"))
    for pkg in ("dense_correspondence", "dense_correspondence/loss_functions", "dense_correspondence/dataset",
                "dense_correspondence/correspondence_tools", "dense_correspondence_manipulation",
                "dense_correspondence_manipulation/utils"):
        _write(os.path.join(pkg, "__init__.py"), "")
    _write("PATCHES.txt", "\n".join(log))
    if verbose:
        print("\n".join(log))
    return OUT


def ref_built():
    return os.path.isfile(os.path.join(OUT, "dense_correspondence", "loss_functions", "loss_composer.py"))


_mods = {}


def load():
    """-> namespace with .pcl (module), .composer (module), .finder (module), .dataset (stub module).
    Imports the generated tree under private names so that it can never shadow the product's compat/ shims."""
    if _mods:
        return _mods["ns"]
    if not ref_built():
        build()
    import importlib
    import types
    import warnings
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in ("dense_correspondence", "dense_correspondence_manipulation")}
    for k in saved:
        del sys.modules[k]
    sys.path.insert(0, OUT)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")          # invalid escape sequences in the reference's docstrings
            ns = types.SimpleNamespace(
                pcl=importlib.import_module("dense_correspondence.loss_functions.pixelwise_contrastive_loss"),
                composer=importlib.import_module("dense_correspondence.loss_functions.loss_composer"),
                finder=importlib.import_module("dense_correspondence.correspondence_tools.correspondence_finder"),
                dataset=importlib.import_module("dense_correspondence.dataset.spartan_dataset_masked"))
    finally:
        sys.path.remove(OUT)
        for k in [k for k in sys.modules if k.split(".")[0] in ("dense_correspondence", "dense_correspondence_manipulation")]:
            del sys.modules[k]
        sys.modules.update(saved)
    _mods["ns"] = ns
    return ns


if __name__ == "__main__":
    print(build(verbose=True))
    ns = load()
    print("imported:", ns.pcl.PixelwiseContrastiveLoss, ns.composer.get_loss, ns.finder.batch_find_pixel_correspondences)
