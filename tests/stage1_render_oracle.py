"""numpy restatements of the stage-1 evaluation kernels: the compose step of render_stage1 at inference (n2m_s1_render_compose,
nerf/renderer.py:886-907) and the viewer's fragment shader on an exported asset (n2m_s1_asset_shade, renderer.html:54-160)."""
import numpy as np


def compose(img, z, bg, h0, w0, ssaa):
    """img [h*w,4] (r, g, b, alpha), z [h*w] (rast's z/w), bg [h0*w0,3] -> image [h0*w0,3], weights_sum [h0*w0], depth [h0*w0] (float64):
    clamp both, alpha * rgb, alpha * z, 2x2 mean (ssaa 2), image + (1 - alpha) * bg"""
    img = np.asarray(img, np.float64).reshape(h0 * ssaa, w0 * ssaa, 4)
    z = np.asarray(z, np.float64).reshape(h0 * ssaa, w0 * ssaa)
    al = np.clip(img[..., 3], 0, 1)
    rgb = al[..., None] * np.clip(img[..., :3], 0, 1)
    dep = al * z

    def mean(x):
        return x.reshape(h0, ssaa, w0, ssaa, *x.shape[2:]).mean(axis=(1, 3))

    rgb, al, dep = mean(rgb), mean(al), mean(dep)
    image = rgb + (1 - al)[..., None] * np.asarray(bg, np.float64).reshape(h0, w0, 3)
    return image.reshape(-1, 3), al.reshape(-1), dep.reshape(-1)


def _bary32(u, v, ww, a0, a1, a2):
    """u a0 + v a1 + (1 - u - v) a2 in float32 with every operation rounded on its own, as the kernel evaluates it"""
    f = np.float32
    return ((f(u) * f(a0)).astype(f) + (f(v) * f(a1)).astype(f)).astype(f) + (f(ww) * f(a2)).astype(f)


def nearest_texel(tex, s, t):
    """three.js NearestFilter + flipY + clamp-to-edge on an RGB uint8 texture [H,W,3]: column clamp(floor(s W)), row clamp(H-1-floor(t H))"""
    H, W = tex.shape[:2]
    x = np.clip(np.floor(np.float32(s) * np.float32(W)).astype(np.int64), 0, W - 1)
    y = np.clip(H - 1 - np.floor(np.float32(t) * np.float32(H)).astype(np.int64), 0, H - 1)
    return tex[y, x]


def specular(w0, w1, x):
    """specular_net in float64: [N,6] -> sigmoid(w1 relu(w0 x)), w0 [32,6], w1 [3,32]"""
    h = np.maximum(np.asarray(x, np.float64) @ np.asarray(w0, np.float64).T, 0)
    return 1 / (1 + np.exp(-(h @ np.asarray(w1, np.float64).T)))


def asset_shade(rast, verts, tri, st, ft, face_offsets, feat0, feat1, w0, w1, campos, mode):
    """rast [n,4] -> img [n,4] (float64): (r, g, b, 1) at covered samples, 0 elsewhere; mode 1 diffuse, 2 specular, 3 full"""
    rast = np.asarray(rast, np.float32).reshape(-1, 4)
    out = np.zeros((rast.shape[0], 4))
    cov = np.nonzero(rast[:, 3] > 0)[0]
    r = rast[cov]
    f = r[:, 3].astype(np.int64) - 1
    cas = np.searchsorted(np.asarray(face_offsets), f, side="right") - 1
    u, v = r[:, 0], r[:, 1]
    ww = (np.float32(1) - u).astype(np.float32) - v
    tf = np.asarray(ft)[f]
    st = np.asarray(st, np.float32)
    s = _bary32(u, v, ww, st[tf[:, 0], 0], st[tf[:, 1], 0], st[tf[:, 2], 0])
    t = _bary32(u, v, ww, st[tf[:, 0], 1], st[tf[:, 1], 1], st[tf[:, 2], 1])
    diffuse = np.zeros((len(cov), 3)); spec_feat = np.zeros((len(cov), 3))
    for c in range(len(feat0)):
        m = cas == c
        diffuse[m] = nearest_texel(np.asarray(feat0[c]), s[m], t[m]) / 255.0
        spec_feat[m] = nearest_texel(np.asarray(feat1[c]), s[m], t[m]) / 255.0
    rgb = diffuse
    if mode != 1:
        vf = np.asarray(tri)[f]
        verts = np.asarray(verts, np.float32)
        x = np.stack([_bary32(u, v, ww, verts[vf[:, 0], a], verts[vf[:, 1], a], verts[vf[:, 2], a]) for a in range(3)], 1).astype(np.float64)
        d = x - np.asarray(campos, np.float64)
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        sp = specular(w0, w1, np.concatenate([d, spec_feat], 1))
        rgb = sp if mode == 2 else np.clip(diffuse + sp, 0, 1)
    out[cov, :3] = rgb
    out[cov, 3] = 1
    return out
