"""Minimal mesh / point-cloud writers for the files the reference's path produces (trimesh is absent here).
  write_off   -- same text layout as source/base/mesh_io.py:79-130 (OFF / COFF)
  write_ply   -- binary little-endian PLY (what trimesh's exporter writes for source/sdf.py:225-228,285)
  read_ply    -- reader for the PLY files this module and trimesh write (ascii or binary_little_endian)
  read_off / read_obj / read_stl -- the other input formats of make_dataset.convert_meshes; read_mesh dispatches
"""
import os

import numpy as np


def make_dir_for_file(path):
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)


def write_off(file_path, vertices, faces, colors_vertex=np.array([]), colors_face=np.array([])):
    vertices = np.asarray(vertices)
    faces = np.asarray(faces)
    colors_vertex = np.asarray(colors_vertex)
    has_vc = colors_vertex.size > 0
    make_dir_for_file(file_path)
    with open(file_path, 'w') as fp:
        fp.write('COFF\n' if has_vc else 'OFF\n')
        fp.write('%d %d 0\n' % (vertices.shape[0], faces.shape[0] if faces.size else 0))
        if has_vc:
            rows = np.concatenate([vertices, colors_vertex], axis=1)
        else:
            rows = vertices
        for r in rows:
            fp.write(' '.join(str(x) for x in r) + '\n')
        if faces.size:
            for f in faces:
                fp.write('3 ' + ' '.join(str(int(i)) for i in f) + '\n')


def write_ply(file_path, vertices, faces=None, colors=None):
    vertices = np.ascontiguousarray(vertices, dtype=np.float32)
    make_dir_for_file(file_path)
    props = [('x', '<f4'), ('y', '<f4'), ('z', '<f4')]
    if colors is not None:
        colors = np.asarray(colors)
        if colors.dtype != np.uint8:
            colors = np.clip(np.round(colors * 255.0), 0, 255).astype(np.uint8)
        props += [('red', 'u1'), ('green', 'u1'), ('blue', 'u1'), ('alpha', 'u1')]
    vrec = np.empty(len(vertices), dtype=props)
    vrec['x'], vrec['y'], vrec['z'] = vertices[:, 0], vertices[:, 1], vertices[:, 2]
    if colors is not None:
        vrec['red'], vrec['green'], vrec['blue'], vrec['alpha'] = colors[:, 0], colors[:, 1], colors[:, 2], 255
    nf = 0 if faces is None else len(faces)
    hdr = ['ply', 'format binary_little_endian 1.0', 'comment points2surf_b200', 'element vertex %d' % len(vertices),
           'property float x', 'property float y', 'property float z']
    if colors is not None:
        hdr += ['property uchar red', 'property uchar green', 'property uchar blue', 'property uchar alpha']
    hdr += ['element face %d' % nf, 'property list uchar int vertex_indices', 'end_header']
    with open(file_path, 'wb') as fp:
        fp.write(('\n'.join(hdr) + '\n').encode('ascii'))
        fp.write(vrec.tobytes())
        if nf:
            frec = np.empty(nf, dtype=[('n', 'u1'), ('v', '<i4', (3,))])
            frec['n'] = 3
            frec['v'] = np.asarray(faces, dtype=np.int32)
            fp.write(frec.tobytes())


def read_ply(file_path):
    """-> (vertices [V,3] float32, faces [F,3] int32 or empty)."""
    with open(file_path, 'rb') as fp:
        header = []
        while True:
            line = fp.readline().decode('ascii', 'replace').strip()
            header.append(line)
            if line == 'end_header':
                break
        fmt = [h for h in header if h.startswith('format')][0].split()[1]
        elems, cur = [], None
        for h in header:
            t = h.split()
            if t and t[0] == 'element':
                cur = {'name': t[1], 'count': int(t[2]), 'props': []}
                elems.append(cur)
            elif t and t[0] == 'property' and cur is not None:
                cur['props'].append(t[1:])
        tmap = {'float': 'f4', 'float32': 'f4', 'double': 'f8', 'float64': 'f8', 'uchar': 'u1', 'uint8': 'u1', 'char': 'i1',
                'int': 'i4', 'int32': 'i4', 'uint': 'u4', 'uint32': 'u4', 'short': 'i2', 'ushort': 'u2'}
        verts, faces = None, np.zeros((0, 3), np.int32)
        if fmt == 'ascii':
            rows = fp.read().decode('ascii').split('\n')
            pos = 0
            for el in elems:
                block = rows[pos:pos + el['count']]
                pos += el['count']
                if el['name'] == 'vertex':
                    names = [p[-1] for p in el['props']]
                    arr = np.array([[float(x) for x in r.split()] for r in block], dtype=np.float64).reshape(el['count'], -1)
                    verts = arr[:, [names.index('x'), names.index('y'), names.index('z')]].astype(np.float32)
                elif el['name'] == 'face' and el['count']:
                    faces = np.array([[int(x) for x in r.split()[1:4]] for r in block], dtype=np.int32)
        else:
            assert fmt == 'binary_little_endian', fmt
            for el in elems:
                if el['count'] == 0:
                    continue
                if el['name'] == 'vertex':
                    dt = np.dtype([(p[-1], '<' + tmap[p[0]]) for p in el['props']])
                    rec = np.frombuffer(fp.read(dt.itemsize * el['count']), dtype=dt)
                    verts = np.stack([rec['x'], rec['y'], rec['z']], axis=1).astype(np.float32)
                elif el['name'] == 'face' and el['count']:
                    p = el['props'][0]
                    assert p[0] == 'list'
                    dt = np.dtype([('n', '<' + tmap[p[1]]), ('v', '<' + tmap[p[2]], (3,))])   # triangles only
                    rec = np.frombuffer(fp.read(dt.itemsize * el['count']), dtype=dt)
                    assert (rec['n'] == 3).all(), 'non-triangular faces'
                    faces = rec['v'].astype(np.int32)
                else:
                    dt = np.dtype([(p[-1], '<' + tmap[p[0]]) for p in el['props']])
                    fp.read(dt.itemsize * el['count'])
    return verts, faces


def _fan(polygons):
    """Polygons (lists of vertex indices) -> triangles [F,3] int32, fans from each polygon's first vertex.  For a quad
    (a, b, c, d) this gives (a, b, c), (a, c, d): the triangles of trimesh's triangulate_quads."""
    tris = [(p[0], p[k], p[k + 1]) for p in polygons for k in range(1, len(p) - 1)]
    return np.array(tris, dtype=np.int32).reshape(-1, 3)


def read_off(file_path):
    """OFF / COFF text files -> (vertices [V,3] float32, faces [F,3] int32); polygon faces are fan-triangulated and
    per-vertex / per-face colours are skipped."""
    with open(file_path) as fp:
        lines = [ln.split('#', 1)[0].split() for ln in fp]
    lines = [t for t in lines if t]
    head = lines[0]
    if not head[0].endswith('OFF'):
        raise ValueError('not an OFF file: %s' % file_path)
    counts = head[1:] if len(head) > 1 else lines[1]
    pos = 1 if len(head) > 1 else 2
    nv, nf = int(counts[0]), int(counts[1])
    verts = np.array([[float(x) for x in t[:3]] for t in lines[pos:pos + nv]], dtype=np.float64).reshape(nv, 3)
    polygons = []
    for t in lines[pos + nv:pos + nv + nf]:
        n = int(t[0])
        polygons.append([int(x) for x in t[1:1 + n]])
    return verts.astype(np.float32), _fan(polygons)


def read_obj(file_path):
    """Wavefront OBJ: `v x y z` and `f` lines (indices as i, i/vt, i//vn or i/vt/vn, 1-based or negative = relative to
    the vertices read so far) -> (vertices [V,3] float32, faces [F,3] int32), polygons fan-triangulated."""
    verts, polygons = [], []
    with open(file_path) as fp:
        for ln in fp:
            t = ln.split()
            if not t:
                continue
            if t[0] == 'v':
                verts.append([float(x) for x in t[1:4]])
            elif t[0] == 'f':
                idx = [int(x.split('/')[0]) for x in t[1:]]
                polygons.append([i - 1 if i > 0 else len(verts) + i for i in idx])
    return np.array(verts, dtype=np.float64).reshape(-1, 3).astype(np.float32), _fan(polygons)


def read_stl(file_path):
    """STL, binary or ASCII -> (vertices [3F,3] float32, faces [F,3] int32): a triangle soup, three vertices per face
    in file order (the clean stage welds them)."""
    with open(file_path, 'rb') as fp:
        data = fp.read()
    if len(data) >= 84:
        n = int(np.frombuffer(data[80:84], '<u4')[0])
        if len(data) == 84 + 50 * n:
            rec = np.frombuffer(data[84:], dtype=[('n', '<f4', (3,)), ('v', '<f4', (3, 3)), ('attr', '<u2')], count=n)
            return rec['v'].reshape(-1, 3).copy(), np.arange(3 * n, dtype=np.int32).reshape(-1, 3)
    text = data.decode('ascii')
    if not text.lstrip().startswith('solid'):
        raise ValueError('not an STL file: %s' % file_path)
    verts = [[float(x) for x in ln.split()[1:4]] for ln in text.split('\n') if ln.strip().startswith('vertex')]
    if len(verts) % 3:
        raise ValueError('STL facet without three vertices: %s' % file_path)
    verts = np.array(verts, dtype=np.float64).reshape(-1, 3).astype(np.float32)
    return verts, np.arange(len(verts), dtype=np.int32).reshape(-1, 3)


def read_mesh(file_path):
    """Dispatch on the extension (.ply / .off / .obj / .stl) -> (vertices, faces)."""
    ext = os.path.splitext(file_path)[1].lower()
    readers = {'.ply': read_ply, '.off': read_off, '.obj': read_obj, '.stl': read_stl}
    if ext not in readers:
        raise ValueError('unsupported mesh format: %s' % file_path)
    return readers[ext](file_path)
