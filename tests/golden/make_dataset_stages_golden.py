"""Write tests/golden/dataset_stages.npz: what the reference's own make_dataset_splits and clean_up_broken_inputs do on
synthetic dataset trees.

    python tests/golden/make_dataset_stages_golden.py REFERENCE_ROOT

The unmodified functions run through oracle/ref_shims.py (trimesh stubbed) with os.listdir returning a fixed,
name-hashed order, so that random.Random(seed).sample sees the same list wherever it runs.  For 3, 10, 37 and 1500
shapes and only_test_set False / True, the npz records the contents of trainset.txt (or its absence), testset.txt and
valset.txt, and the files clean_up_broken_inputs moved.  tests/test_mesh_clean_host.py builds the same trees
(make_tree) and runs this repository's mirrors under the same listdir order."""
import contextlib
import hashlib
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SIZES = (3, 10, 37, 1500)
CLEAN_UP_DIRS = ['03_meshes', '04_pts', '05_query_pts', '05_query_dist', 'not_there']


def shape_names(n):
    return ['%08d_%s' % (i * 7919 % 100000000, hashlib.md5(str(i).encode()).hexdigest()[:12]) for i in range(n)]


def make_tree(base, n):
    """dataset 'ds' under base: every shape in 03_meshes, 04_pts and 05_query_pts; every third shape lacks its
    05_query_dist file, which holds a stray .txt instead."""
    names = shape_names(n)
    files = {'03_meshes': '%s.ply', '04_pts': '%s.xyz.npy', '05_query_pts': '%s.ply.npy'}
    for d, pattern in files.items():
        os.makedirs(os.path.join(base, 'ds', d), exist_ok=True)
        for s in names:
            open(os.path.join(base, 'ds', d, pattern % s), 'w').close()
    os.makedirs(os.path.join(base, 'ds', '05_query_dist', 'subdir'), exist_ok=True)
    for i, s in enumerate(names):
        name = s + ('.txt' if i % 3 == 0 else '.ply.npy')
        open(os.path.join(base, 'ds', '05_query_dist', name), 'w').close()


@contextlib.contextmanager
def fixed_listdir():
    """os.listdir in ascending MD5 order of the names: fixed, and unlike both sorted and file-system order."""
    real = os.listdir

    def listdir(path='.'):
        return sorted(real(path), key=lambda s: hashlib.md5(s.encode()).hexdigest())
    os.listdir = listdir
    try:
        yield
    finally:
        os.listdir = real


def run_case(make_dataset_splits, clean_up_broken_inputs, n, only_test_set):
    """-> dict of the recorded outputs for one tree."""
    with tempfile.TemporaryDirectory() as base, fixed_listdir():
        make_tree(base, n)
        make_dataset_splits(base, 'ds', '05_query_pts', seed=42, only_test_set=only_test_set, testset_ratio=0.1)
        clean_up_broken_inputs(base, 'ds', '05_query_dist', '.npy', CLEAN_UP_DIRS, broken_dir='broken')
        out = {}
        for split in ('trainset', 'testset', 'valset'):
            p = os.path.join(base, 'ds', split + '.txt')
            out[split] = open(p).read() if os.path.exists(p) else '<missing>'
        moved = []
        for root, _, files in os.walk(os.path.join(base, 'ds', 'broken')):
            moved += [os.path.relpath(os.path.join(root, f), os.path.join(base, 'ds')) for f in files]
        out['moved'] = '\n'.join(sorted(moved))
        return out


def main(ref_root):
    sys.path.insert(0, ROOT)
    from oracle import ref_shims
    ref_shims.REFERENCE_ROOT = ref_root
    ref_shims.install()
    for m in [m for m in sys.modules if m == 'source' or m.startswith('source.')]:
        del sys.modules[m]          # this repository's source/ shim package must not shadow the reference's
    sys.path.remove(ROOT)
    sys.path.insert(0, ref_root)
    import make_dataset as ref_md
    assert os.path.dirname(os.path.abspath(ref_md.__file__)) == os.path.abspath(ref_root)
    out = {}
    for n in SIZES:
        for ots in (False, True):
            rec = run_case(ref_md.make_dataset_splits, ref_md.clean_up_broken_inputs, n, ots)
            for k, val in rec.items():
                out['%s_%d_%d' % (k, n, ots)] = np.array(val)
            print(n, ots, 'test', len(rec['testset'].split('\n')), 'moved', len(rec['moved'].split('\n')))
    path = os.path.join(ROOT, 'tests', 'golden', 'dataset_stages.npz')
    np.savez_compressed(path, **out)
    print('written', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main(sys.argv[1])
