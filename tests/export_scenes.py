"""Scenes for the colour plan (tests/test_oracle_export.py, tests/test_gpu_export.py, scripts/bench_export.py) and a
plain-Python restatement of Regard3D's ColorizeTracks loop to hold the oracle to.

A scene is (views, landmarks) in the shape SfmData.views() / SfmData.landmarks() return: views as dicts with id_view,
width, height and has_pose; landmarks as dicts with id, X and obs = [(id_view, id_feat, x, y), ...] in view order."""
import numpy as np


def random_scene(seed, n_views=12, n_lm=300, max_obs=4, posed_frac=0.75, edge_frac=0.3, sizes=((64, 48), (5, 3), (640, 480))):
    """Views with ids spread out, a share of them (the last one always) without a pose and never observed, as after the
    engine; landmarks with 1..max_obs observations in posed views, a share of the coordinates in (-1, 0) or [w - 1, w).
    Few posed views and small tracks make equal per-view counts common, so the tie rule decides many rounds."""
    rng = np.random.default_rng(seed)
    ids = np.sort(rng.choice(10 * n_views, n_views, replace=False)).astype(np.uint32)
    views = []
    for k, v in enumerate(ids.tolist()):
        w, h = sizes[rng.integers(len(sizes))]
        views.append(dict(id_view=v, width=w, height=h, has_pose=bool(k == 0 or (k < n_views - 1 and rng.random() < posed_frac))))
    posed = [v for v in views if v["has_pose"]]
    lm_ids = np.sort(rng.choice(10 * n_lm, n_lm, replace=False)).astype(np.uint32)
    landmarks = []
    for l in lm_ids.tolist():
        k = int(rng.integers(1, min(max_obs, len(posed)) + 1))
        vs = sorted(rng.choice(len(posed), k, replace=False).tolist(), key=lambda i: posed[i]["id_view"])
        obs = []
        for i in vs:
            v = posed[i]
            xy = []
            for size in (v["width"], v["height"]):
                u = rng.random()
                if u < edge_frac / 2:
                    xy.append(float(-rng.uniform(0.0, 1.0)) if rng.random() < 0.9 else -0.9999999999)
                elif u < edge_frac:
                    xy.append(float(size - 1 + rng.uniform(0.0, 1.0)) if rng.random() < 0.9 else size - 1e-10)
                else:
                    xy.append(float(rng.uniform(0.0, size - 1)))
            obs.append((v["id_view"], int(rng.integers(1000)), xy[0], xy[1]))
        landmarks.append(dict(id=l, X=rng.normal(size=3).tolist(), obs=obs))
    return views, landmarks


def ba_scene(n_cams=100, n_pts=100000, obs_per_pt=5, seed=29, twins=True, w=1920, h=1080):
    """The bundle-adjustment problem generator's scene (synth.make_ba_problem) as views and landmarks; with twins, each
    view has a twin that observes exactly what it observes at the same pixel, so every round starts with a forced tie
    that the twin of lower id wins."""
    from regard3d_b200 import synth
    p = synth.make_ba_problem(n_cams=n_cams, n_pts=n_pts, obs_per_pt=obs_per_pt, seed=seed, w=w, h=h)
    n_lm = len(p["points"])
    xy = p["obs_xy"].reshape(n_lm, obs_per_pt, 2).copy()
    xy[..., 0] = np.clip(xy[..., 0], -0.5, w - 0.5)
    xy[..., 1] = np.clip(xy[..., 1], -0.5, h - 0.5)
    cam = p["obs_cam"].reshape(n_lm, obs_per_pt)
    n_views = 2 * n_cams if twins else n_cams
    views = [dict(id_view=v, width=w, height=h, has_pose=True) for v in range(n_views)]
    landmarks = []
    for l in range(n_lm):
        obs = [(int(c), l, float(xy[l, k, 0]), float(xy[l, k, 1])) for k, c in enumerate(cam[l].tolist())]
        if twins:
            obs += [(n_cams + c, f, x, y) for (c, f, x, y) in obs]
        landmarks.append(dict(id=l, X=p["points"][l].tolist(), obs=sorted(obs)))
    return views, landmarks


def python_plan(views, landmarks):
    """ColorizeTracks restated with dicts and sets: (round_view, lm_round, lm_pixel) with landmarks in id order."""
    lms = {l["id"]: {o[0]: (o[2], o[3]) for o in l["obs"]} for l in landmarks}
    order = sorted(lms)
    index = {t: i for i, t in enumerate(order)}
    remaining = set(order)
    round_view, lm_round, lm_pixel = [], [0] * len(order), [(0, 0)] * len(order)
    while remaining:
        card = {}
        for t in remaining:
            for v in lms[t]:
                card[v] = card.get(v, 0) + 1
        best = max(card.values())
        view = min(v for v, c in card.items() if c == best)
        colored = [t for t in remaining if view in lms[t]]
        for t in colored:
            x, y = lms[t][view]
            lm_round[index[t]] = len(round_view)
            lm_pixel[index[t]] = (int(x), int(y))  # truncation toward zero, as the image index conversion
        remaining.difference_update(colored)
        round_view.append(view)
    return (np.array(round_view, np.uint32), np.array(lm_round, np.uint32),
            np.array(lm_pixel, np.int32).reshape(-1, 2))


def to_sfm(capi, views, landmarks, model=3):
    """The scene as an SfmData: one intrinsic per view size, a pose for every view that has one."""
    sd = capi.SfmData()
    sizes = sorted({(v["width"], v["height"]) for v in views})
    for i, (w, h) in enumerate(sizes):
        sd.add_intrinsic(i, model, w, h, 1.2 * max(w, h), w / 2.0, h / 2.0, (0.0, 0.0, 0.0))
    for v in views:
        vid = v["id_view"]
        sd.add_view(vid, "image%06d.jpg" % vid, v["width"], v["height"], id_intrinsic=sizes.index((v["width"], v["height"])),
                    id_pose=vid if v["has_pose"] else 1 << 30)
        if v["has_pose"]:
            sd.add_pose(vid, np.eye(3), [0.01 * vid, 0.0, 0.0])
    for l in landmarks:
        sd.add_landmark(l["id"], l["X"], l["obs"])
    return sd


def oracle_plan(views, landmarks):
    from oracle import pyoracle_export as pe
    return pe.colorize_plan(*pe.flatten(views, landmarks))


def image_for(view_id, w, h):
    """A deterministic RGB image per view id."""
    rng = np.random.default_rng(1000 + view_id)
    return rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
