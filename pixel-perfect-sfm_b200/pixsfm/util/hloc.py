"""hloc-side inputs of the keypoint adjustment (reference pixsfm/util/hloc.py:11-70): the image-pair list (text) and
the keypoint / match files hloc writes (HDF5), through h5py when present and util/h5lite.py otherwise."""
import numpy as np


def read_image_pairs(path):
    """one "name1 name2" pair per line -> [[name1, name2], ...]"""
    with open(path) as f:
        return [line.split() for line in f.read().splitlines() if line.strip()]


def write_image_pairs(path, pairs):
    with open(path, "w") as f:
        f.write("\n".join("%s %s" % (a, b) for a, b in pairs))


def matches_from_hloc_arrays(matches0, scores0=None, reverse=False):
    """hloc stores, per keypoint of the first image, the index of its match in the second (-1: none) and a score.
    -> (matches uint64 [M,2], scores float32 [M] or None); `reverse` swaps the columns when the pair is stored as
    (second, first)"""
    matches0 = np.asarray(matches0).reshape(-1)
    first = np.flatnonzero(matches0 != -1)
    pairs = np.stack([first, matches0[first]], axis=-1).astype(np.uint64)
    if reverse:
        pairs = pairs[:, ::-1].copy()
    scores = None if scores0 is None else np.asarray(scores0).reshape(-1)[first].astype(np.float32)
    return pairs, scores


def _h5py():
    """h5py when it is installed, else the built-in reader/writer of the classic HDF5 layout (util/h5lite.py: what h5py
    writes by default and hloc's files use)"""
    try:
        import h5py
        return h5py
    except ImportError:
        from . import h5lite
        return h5lite


def _pair_key(h5f, name1, name2):
    """hloc.utils.io.find_pair: the group of a pair under either order and either separator -> (key, reversed)"""
    def flat(name):
        return name.replace("/", "-")
    for key, rev in ((flat(name1) + "/" + flat(name2), False), (flat(name2) + "/" + flat(name1), True),
                     (flat(name1) + "_" + flat(name2), False), (flat(name2) + "_" + flat(name1), True)):
        if key in h5f:
            return key, rev
    raise ValueError("Could not find pair %s %s in the match file" % (name1, name2))


def list_h5_names(path):
    h5py = _h5py()
    found = set()
    with h5py.File(str(path), "r") as f:
        f.visititems(lambda _, obj: found.add(obj.parent.name.strip("/")) if isinstance(obj, h5py.Dataset) else None)
    return sorted(found)


def read_keypoints_hloc(path, names=None, as_cpp_map=False):
    h5py = _h5py()
    names = list_h5_names(path) if names is None else names
    with h5py.File(str(path), "r") as f:
        return {name: np.asarray(f[name]["keypoints"])[:, :2].astype(np.float64) for name in names}


def read_keypoint_uncertainty(path, names):
    """{name: the `uncertainty` attribute of the image's keypoint dataset, or None}: the keypoint noise in pixels that
    hloc's feature extraction records (hloc.utils.io.get_keypoints(..., return_uncertainty=True))"""
    h5py = _h5py()
    with h5py.File(str(path), "r") as f:
        out = {}
        for name in names:
            u = f[name]["keypoints"].attrs.get("uncertainty")
            out[name] = None if u is None else float(np.asarray(u).reshape(-1)[0])
        return out


def write_keypoints_hloc(path, keypoint_dict):
    h5py = _h5py()
    with h5py.File(str(path), "w") as f:
        for name, keypoints in keypoint_dict.items():
            f.create_group(name).create_dataset("keypoints", data=keypoints)


def read_matches_hloc(path, pairs):
    h5py = _h5py()
    matches, scores = [], []
    with h5py.File(str(path), "r") as f:
        for name1, name2 in pairs:
            key, reverse = _pair_key(f, str(name1), str(name2))
            m, s = matches_from_hloc_arrays(np.asarray(f[key]["matches0"]), np.asarray(f[key]["matching_scores0"]), reverse)
            matches.append(m); scores.append(s)
    return matches, scores
