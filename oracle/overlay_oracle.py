"""TEST INFRASTRUCTURE — CPU restatement of the target preparation (src/preparation.py:18-198); only tests/ and
oracle/make_golden_overlay.py import it.

  * `rle_fr_poly` / `decode` / `fr_py_objects` / `merge`: pycocotools' maskApi.c rleFrPoly, rleDecode and rleMerge
    (the published algorithm behind cocomask.frPyObjects + decode), restated in numpy.  No implementation of it exists
    where the tests run, so tests/test_overlay_cpu.py pins it with vectors derived by hand from maskApi.c and with the
    property that an integer axis-aligned box rasterises to exactly [x0, x1) x [y0, y1), clipped to the image.
  * `binary_erosion` / `binary_dilation` / `rectangle`: skimage <= 0.17, which call
    ndi.binary_erosion(structure=selem, border_value=True) and ndi.binary_dilation(structure=selem) -- an assumption
    about the skimage version the reference ran, like DESIGN.md section 3's for skimage.transform.resize.
  * `overlay_mask_one_image`: the reference's per-image function on an annotation list, returning instead of writing.
    Distances and sizes reuse oracle/input_oracle.py.
"""
import numpy as np
from scipy import ndimage as ndi

from . import input_oracle as IO

SCALE = 5.0
INT_MIN = -2 ** 31


def _trunc_int(a):
    """C's (int) of a double: truncation toward zero; x86 cvttsd2si turns NaN into INT_MIN"""
    a = np.asarray(a, np.float64)
    out = np.full(a.shape, INT_MIN, np.int64)
    ok = ~np.isnan(a)
    out[ok] = np.trunc(a[ok]).astype(np.int64)
    return out


def scaled_vertices(poly):
    """(int)(5 x + .5) of every coordinate, checked to fit C's int -> (x int64 [k], y int64 [k])"""
    xy = np.asarray(poly, np.float64)
    k = len(xy) // 2
    xy = xy[:2 * k]
    s = _trunc_int(np.float64(SCALE) * xy + 0.5)
    if np.isnan(xy).any() or (s < INT_MIN + 1).any() or (s > 2 ** 31 - 1).any():
        raise ValueError("polygon vertex out of range: 5 * coordinate must fit a 32-bit int")
    return s[0::2], s[1::2]


def boundary_points(poly):
    """rleFrPoly's dense walk of the closed polygon: -> (u, v) int64 over all edges, concatenated"""
    x, y = scaled_vertices(poly)
    k = len(x)
    us, vs = [], []
    for j in range(k):
        xs, ys, xe, ye = int(x[j]), int(y[j]), int(x[(j + 1) % k]), int(y[(j + 1) % k])
        dx, dy = abs(xe - xs), abs(ys - ye)
        flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
        if flip:
            xs, xe, ys, ye = xe, xs, ye, ys
        if dx >= dy:
            t = np.arange(dx + 1, dtype=np.int64)
            t = dx - t if flip else t
            s = np.float64(ye - ys) / np.float64(dx) if dx else np.float64(np.nan)
            us.append(t + xs)
            vs.append(_trunc_int((np.float64(ys) + s * t.astype(np.float64)) + 0.5))
        else:
            t = np.arange(dy + 1, dtype=np.int64)
            t = dy - t if flip else t
            s = np.float64(xe - xs) / np.float64(dy)
            vs.append(t + ys)
            us.append(_trunc_int((np.float64(xs) + s * t.astype(np.float64)) + 0.5))
    if not us:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(us), np.concatenate(vs)


def toggle_positions(poly, h, w):
    """the column-major positions x * h + y of rleFrPoly's column crossings (before the sort)"""
    u, v = boundary_points(poly)
    if len(u) < 2:
        return np.zeros(0, np.int64)
    j = np.nonzero(u[1:] != u[:-1])[0] + 1
    uj, up, vj, vp = u[j], u[j - 1], v[j], v[j - 1]
    xd = (np.where(uj < up, uj, uj - 1).astype(np.float64) + 0.5) / SCALE - 0.5
    keep = (np.floor(xd) == xd) & (xd >= 0) & (xd <= w - 1)
    yd = (np.minimum(vj, vp).astype(np.float64) + 0.5) / SCALE - 0.5
    yd = np.ceil(np.clip(yd, 0, h))
    return xd[keep].astype(np.int64) * h + yd[keep].astype(np.int64)


def rle_fr_poly(poly, h, w):
    """RLE counts (uint32 list) of one polygon, as rleFrPoly builds them"""
    a = np.sort(np.append(toggle_positions(poly, h, w), h * w))
    d = np.diff(np.concatenate([[0], a]))
    b = [int(d[0])]
    j = 1
    while j < len(d):
        if d[j] > 0:
            b.append(int(d[j]))
            j += 1
        else:
            j += 1
            if j < len(d):
                b[-1] += int(d[j])
                j += 1
    return b


def decode(counts, h, w):
    """rleDecode -> uint8 (h, w)"""
    flat = np.zeros(h * w, np.uint8)
    p, v = 0, 0
    for c in counts:
        flat[p:p + c] = v
        p += c
        v ^= 1
    return flat.reshape(w, h).T.copy()


def encode(mask):
    """canonical COCO counts of a (h, w) mask (column-major runs, zeros first)"""
    flat = np.asarray(mask, np.uint8).T.reshape(-1)
    change = np.nonzero(np.diff(flat))[0] + 1
    edges = np.concatenate([[0], change, [flat.size]])
    runs = np.diff(edges).tolist()
    return ([0] + runs) if flat.size and flat[0] else runs


def polygon_mask(poly, h, w):
    return decode(rle_fr_poly(poly, h, w), h, w)


def segmentation_form(segm):
    """which frPyObjects branch a COCO segmentation takes: 'polygons', 'bbox' or 'RLE'"""
    if isinstance(segm, dict):
        return "RLE"
    if isinstance(segm, (list, tuple)) and len(segm) and isinstance(segm[0], (list, tuple, np.ndarray)):
        if len(segm[0]) < 4:
            return "unsupported"
        return "bbox" if len(segm[0]) == 4 else "polygons"
    if isinstance(segm, (list, tuple)) and len(segm) and isinstance(segm[0], dict):
        return "RLE"
    if isinstance(segm, (list, tuple)) and not len(segm):
        return "unsupported"
    if isinstance(segm, (list, tuple)) and len(segm) == 4:
        return "bbox"
    return "flat polygon" if isinstance(segm, (list, tuple)) else "unknown"


def fr_py_objects(segm, h, w):
    """frPyObjects for a list of polygons -> list of RLE counts"""
    form = segmentation_form(segm)
    if form == "unsupported":
        raise ValueError("segmentation input type is not supported")   # pycocotools raises a bare Exception
    if form != "polygons":
        raise NotImplementedError("only COCO polygon segmentations are rasterised, not the %s form" % form)
    return [rle_fr_poly(p, h, w) for p in segm]


def decode_stack(rles, h, w):
    """cocomask.decode of a list of RLEs -> uint8 (h, w, n), Fortran-ordered as pycocotools returns it"""
    if not rles:
        return np.zeros((h, w, 0), np.uint8, order="F")
    return np.asfortranarray(np.stack([decode(r, h, w) for r in rles], axis=2))


def merge(rles, h, w):
    """rleMerge (union): a single RLE is returned as is"""
    if len(rles) == 1:
        return list(rles[0])
    m = np.zeros((h, w), np.uint8)
    for r in rles:
        m |= decode(r, h, w)
    return encode(m)


def ann_to_rle(segm, h, w):
    """COCO.annToRLE of a polygon segmentation: merge(frPyObjects(segm, h, w))"""
    return merge(fr_py_objects(segm, h, w), h, w)


# ---------------------------------------------------------------------------------------------------------------------
# skimage <= 0.17 binary morphology
# ---------------------------------------------------------------------------------------------------------------------
def rectangle(width, height, dtype=np.uint8):
    return np.ones((width, height), dtype=dtype)


def binary_erosion(image, selem=None):
    return ndi.binary_erosion(image, structure=selem, border_value=True)


def binary_dilation(image, selem=None):
    return ndi.binary_dilation(image, structure=selem)


# ---------------------------------------------------------------------------------------------------------------------
# overlay_mask_one_image
# ---------------------------------------------------------------------------------------------------------------------
def _on_border(m, b):
    return not np.any(m[b:-b, b:-b])


def _instances(annotations, h, w, erode, dilate, small_annotations_size):
    """the instance masks of one category in the reference's order -> (full-mask instances, distance instances)"""
    full, dist = [], []
    for ann in annotations:
        m = decode_stack(fr_py_objects(ann["segmentation"], h, w), h, w)
        if erode == 0:
            for i in range(m.shape[-1]):
                mi = m[:, :, i]
                if not _on_border(mi, 2):
                    full.append(mi)
                    dist.append(mi)
            continue
        for i in range(m.shape[-1]):
            if not _on_border(m[:, :, i], 2):
                full.append(m[:, :, i])
        if m.shape[-1] != 1:
            raise ValueError("an annotation with %d polygons cannot be eroded as one mask" % m.shape[-1])
        mi = m[:, :, 0]
        if _on_border(mi, 2):
            continue
        if mi.sum() > small_annotations_size ** 2:
            mi = binary_erosion(mi, rectangle(erode, erode))
        elif dilate > 0:
            mi = binary_dilation(mi, rectangle(dilate, dilate))
        dist.append(np.asarray(mi, np.uint8))
    return full, dist


def _union(planes, h, w):
    m = np.zeros((h, w), np.uint8)
    for p in planes:
        m |= (p != 0)
    return m


def add_dropped_objects(original, processed):
    """src/utils.py:333-339"""
    out = processed.copy()
    lab, k = ndi.label(original)
    for i in range(1, k + 1):
        comp = lab == i
        if not np.any(comp & (processed != 0)):
            out = out + comp
    return out.astype(np.uint8)


def overlay_mask_one_image(annotations, h, w, category_ids=(None, 100), erode=0, dilate=0, border_width=0,
                           small_annotations_size=14):
    """src/preparation.py:44-100 for one image whose annotations (file order) are given ->
    (mask uint8, distances float16, sizes (int64, or uint8 ones without any component))"""
    mask = np.zeros((h, w), np.uint8)
    dist = np.zeros((h, w))
    for nr, cid in enumerate(category_ids):
        if cid is None:
            continue
        if erode < 0 or dilate < 0:
            raise ValueError("erode and dilate cannot be negative")
        anns = [a for a in annotations if a["category_id"] == cid]
        full, inst = _instances(anns, h, w, erode, dilate, small_annotations_size)
        for m in inst:
            dist = IO.update_distances(dist, m)
        if erode > 0 and dilate == 0:
            m = add_dropped_objects(_union(full, h, w), _union(inst, h, w))
        else:
            m = _union(inst, h, w)
        mask = np.where(m, nr, mask).astype(np.uint8)
    sizes = IO.get_size_matrix(mask)
    dist16, second = IO.clean_distances(dist)
    if border_width > 0:
        borders = (second < border_width) & (~mask)
        mask = np.where(borders, mask.max() + 1, mask).astype(np.uint8)
    return mask, dist16, sizes


# ---------------------------------------------------------------------------------------------------------------------
# seeded synthetic annotations
# ---------------------------------------------------------------------------------------------------------------------
def _rotate(pts, cx, cy, theta):
    c, s = np.cos(theta), np.sin(theta)
    x, y = pts[:, 0], pts[:, 1]
    return np.stack([cx + c * x - s * y, cy + s * x + c * y], axis=1)


def building_polygon(rs, h, w, size=None, center=None):
    """one building-like polygon with float vertices: a rotated rectangle, an L-shape or a convex n-gon"""
    a = float(size if size is not None else rs.choice([rs.uniform(2, 7), rs.uniform(8, 25), rs.uniform(26, 70)]))
    b = a * rs.uniform(0.4, 1.0)
    cx, cy = center if center is not None else (rs.uniform(-0.1 * w, 1.1 * w), rs.uniform(-0.1 * h, 1.1 * h))
    kind = rs.randint(3)
    if kind == 0:
        pts = np.array([[-a, -b], [a, -b], [a, b], [-a, b]]) / 2
    elif kind == 1:
        pts = np.array([[-a, -b], [a, -b], [a, 0], [0, 0], [0, b], [-a, b]]) / 2
    else:
        ang = np.sort(rs.uniform(0, 2 * np.pi, rs.randint(3, 9)))
        pts = np.stack([a / 2 * np.cos(ang), b / 2 * np.sin(ang)], axis=1)
    pts = _rotate(pts, cx, cy, rs.uniform(0, np.pi))
    if rs.rand() < 0.5:
        pts = pts[::-1]
    return [round(float(v), 2) for v in pts.reshape(-1)]


def eroded_to_empty(annotations, h, w, erode, small_annotations_size=14):
    """how many kept annotations the erosion branch empties (their distance transform is scipy's no-background one)"""
    if erode <= 0:
        return 0
    count = 0
    for ann in annotations:
        m = polygon_mask(ann["segmentation"][0], h, w)
        if not _on_border(m, 2) and m.sum() > small_annotations_size ** 2:
            count += not binary_erosion(m, rectangle(erode, erode)).any()
    return count


def synthetic_image_annotations(rs, h, w, n_buildings, image_id, first_ann_id, multi_polygon=True, category_id=100):
    """COCO annotations of one image: buildings of all sizes, some overlapping, touching or crossing the border or wholly
    outside it, thin ones that erode to nothing, multi-polygon annotations (when allowed) and, now and then, a
    whole-image polygon first"""
    anns = []
    for k in range(n_buildings):
        r = rs.rand()
        if k == 0 and r < 0.1:
            segm = [[-1.0, -1.0, w + 1.0, -1.0, w + 1.0, h + 1.0, -1.0, h + 1.0]]
        elif r < 0.2:
            # thin: at most 2 rows and, on a 300 x 300 image, over the 14 ** 2 erosion gate, so a 3 x 3 erosion
            # empties it (on the small images it is clipped under the gate)
            t = rs.uniform(1.0, 2.0)
            x0, y0, ln = rs.uniform(3, max(w - 265, 4)), rs.uniform(3, h - 5), rs.uniform(200, 260)
            segm = [[x0, y0, x0 + ln, y0, x0 + ln, y0 + t, x0, y0 + t]]
        elif r < 0.25:
            segm = [building_polygon(rs, h, w, center=(rs.uniform(w + 5, w + 60), rs.uniform(-60, h + 60)))]
        elif r < 0.33 and anns:
            prev = np.asarray(anns[-1]["segmentation"][0]).reshape(-1, 2).mean(0)   # overlaps the previous one
            segm = [building_polygon(rs, h, w, center=tuple(prev + rs.uniform(-5, 5, 2)))]
        elif r < 0.43 and multi_polygon:
            segm = [building_polygon(rs, h, w) for _ in range(rs.randint(2, 4))]
        else:
            segm = [building_polygon(rs, h, w)]
        segm = [[round(float(v), 2) for v in p] for p in segm]
        anns.append({"id": first_ann_id + k, "image_id": image_id, "category_id": category_id, "segmentation": segm,
                     "iscrowd": 0, "area": 1.0, "bbox": [0.0, 0.0, 1.0, 1.0]})
    return anns
