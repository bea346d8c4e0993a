"""CPU tests of the WebXR view rectangles of SplatScene.render_xr_views: native XRWebGLLayer.getViewport(view) rectangles
scaled by xrPixelRatio and floored, component by component, as render_xr sizes its eyes."""
import importlib

gs = importlib.import_module("aframe-gaussian-splatting_b200")


def test_side_by_side_eyes_match_render_xr_layer():
    """Two native 1832 x 1920 eyes at xrPixelRatio 0.5: the rectangles render_xr_layer draws, (0, 0) and (w, 0)."""
    assert gs.component.xr_viewports([(0, 0, 1832, 1920), (1832, 0, 1832, 1920)], 0.5) == [(0, 0, 916, 960), (916, 0, 916, 960)]


def test_every_component_floored():
    ratio = 0.7
    got = gs.component.xr_viewports([(3, 5, 97, 95), (1, 1, 1, 1), (2561, 0, 1281, 721)], ratio)
    assert got == [(2, 3, 67, 66), (0, 0, 0, 0), (1792, 0, 896, 504)]
    for vp, r in zip([(3, 5, 97, 95), (1, 1, 1, 1), (2561, 0, 1281, 721)], got):
        assert all(isinstance(c, int) and c == int(v * ratio // 1) for c, v in zip(r, vp))


def test_ratio_one_keeps_native_rectangles():
    vps = [(0, 0, 916, 960), (916, 0, 916, 960), (1832, 0, 1280, 720), (0, 960, 640, 640)]
    assert gs.component.xr_viewports(vps, 1.0) == vps
