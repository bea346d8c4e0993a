// UNBUILT SOURCE: this image has no Node toolchain (node, npm, node_api.h are absent).  It shows the N-API
// addon a maintainer of the reference would add to bind include/gsplat_b200.h; see INTEGRATION.md.
// bindings/node/gsplat_napi.cc  —  node-gyp: link -lgsplat_b200, include ../../include
#include <napi.h>
#include <cstring>
#include <vector>
#include "gsplat_b200.h"

class Splats : public Napi::ObjectWrap<Splats> {
 public:
  static Napi::Object Init(Napi::Env env, Napi::Object exports) {
    exports.Set("Splats", DefineClass(env, "Splats", {
      InstanceMethod("clear", &Splats::Clear), InstanceMethod("push", &Splats::Push),
      InstanceMethod("pushPly", &Splats::PushPly), InstanceMethod("reserve", &Splats::Reserve),
      InstanceMethod("sort", &Splats::Sort),   InstanceMethod("render", &Splats::Render),
      InstanceMethod("renderScene", &Splats::RenderScene), InstanceMethod("insert", &Splats::Insert),
      InstanceMethod("insertPly", &Splats::InsertPly), InstanceMethod("erase", &Splats::Erase),
      InstanceMethod("renderSceneXR", &Splats::RenderSceneXR), InstanceMethod("pickScene", &Splats::PickScene)}));
    // the RGBA8 target's per-fragment rounding: frame objects take `blendUnorm8: true` (GS_RENDER_BLEND_UNORM8)
    exports.Set("BLEND_UNORM8", Napi::Number::New(env, GS_RENDER_BLEND_UNORM8));
    return exports;
  }
  explicit Splats(const Napi::CallbackInfo& i) : Napi::ObjectWrap<Splats>(i) {
    int dev = i.Length() ? i[0].As<Napi::Number>().Int32Value() : 0;
    if (gs_create(dev, &ctx_) != GS_OK) Napi::Error::New(i.Env(), gs_last_error(nullptr)).ThrowAsJavaScriptException();
  }
  ~Splats() { gs_destroy(ctx_); }
 private:
  void Check(Napi::Env e, int rc) { if (rc != GS_OK) Napi::Error::New(e, gs_last_error(ctx_)).ThrowAsJavaScriptException(); }
  // {blendUnorm8: true}: the bytes the page's RGBA8 framebuffer holds after the reference's blend, rounded per fragment
  static uint32_t Blend8(const Napi::Object& o) {
    return (o.Has("blendUnorm8") && o.Get("blendUnorm8").ToBoolean().Value()) ? (uint32_t)GS_RENDER_BLEND_UNORM8 : 0u;
  }
  Napi::Value Clear(const Napi::CallbackInfo& i) { Check(i.Env(), gs_clear(ctx_)); return i.Env().Undefined(); }
  // reserve(numVertexes)                           <- initGL(numVertexes), index.js:248-251
  Napi::Value Reserve(const Napi::CallbackInfo& i) {
    Check(i.Env(), gs_reserve(ctx_, i[0].As<Napi::Number>().Uint32Value()));
    return i.Env().Undefined();
  }
  // push(ArrayBuffer rows, vertexCount)            <- pushDataBuffer(buffer, vertexCount), index.js:328
  Napi::Value Push(const Napi::CallbackInfo& i) {
    auto buf = i[0].As<Napi::ArrayBuffer>();
    Check(i.Env(), gs_push_splats(ctx_, buf.Data(), i[1].As<Napi::Number>().Uint32Value()));
    return i.Env().Undefined();
  }
  // pushPly(ArrayBuffer plyFile) -> vertexCount    <- processPlyBuffer + pushDataBuffer, index.js:315-324, 600-745
  Napi::Value PushPly(const Napi::CallbackInfo& i) {
    auto buf = i[0].As<Napi::ArrayBuffer>();
    uint32_t n = 0;
    Check(i.Env(), gs_push_ply(ctx_, buf.Data(), buf.ByteLength(), nullptr, &n));
    return Napi::Number::New(i.Env(), n);
  }
  // insert(at, ArrayBuffer rows, vertexCount)     <- one entity's pushDataBuffer into the shared table, at the end of its
  //                                                   own range: entities stream in together (index.js:259-298)
  Napi::Value Insert(const Napi::CallbackInfo& i) {
    auto buf = i[1].As<Napi::ArrayBuffer>();
    Check(i.Env(), gs_insert_splats(ctx_, i[0].As<Napi::Number>().Uint32Value(), buf.Data(),
                                    i[2].As<Napi::Number>().Uint32Value()));
    return i.Env().Undefined();
  }
  // insertPly(at, ArrayBuffer plyFile) -> vertexCount   <- pushPly into one entity's range
  Napi::Value InsertPly(const Napi::CallbackInfo& i) {
    auto buf = i[1].As<Napi::ArrayBuffer>();
    uint32_t n = 0;
    Check(i.Env(), gs_insert_ply(ctx_, i[0].As<Napi::Number>().Uint32Value(), buf.Data(), buf.ByteLength(), nullptr, &n));
    return Napi::Number::New(i.Env(), n);
  }
  // erase(first, count)                            <- one entity's worker "clear" (index.js:236,573-575) in a shared table
  Napi::Value Erase(const Napi::CallbackInfo& i) {
    Check(i.Env(), gs_erase(ctx_, i[0].As<Napi::Number>().Uint32Value(), i[1].As<Napi::Number>().Uint32Value()));
    return i.Env().Undefined();
  }
  // sort(Float32Array view, Float32Array|undefined cutout) -> Uint32Array   <- worker "sort", index.js:587-596
  Napi::Value Sort(const Napi::CallbackInfo& i) {
    auto view = i[0].As<Napi::Float32Array>();
    const float* cut = i[1].IsUndefined() ? nullptr : i[1].As<Napi::Float32Array>().Data();
    uint32_t n = 0, cnt = 0; gs_num_splats(ctx_, &n);
    auto out = Napi::Uint32Array::New(i.Env(), n);
    Check(i.Env(), gs_sort(ctx_, view.Data(), cut, out.Data(), &cnt));
    return Napi::Uint32Array::New(i.Env(), cnt, out.ArrayBuffer(), 0);
  }
  // render({proj, modelview, width, height, focal, cutout?, bg?, depth?: Float32Array, blendUnorm8?}, Uint8Array out)
  //                                                <- onBeforeRender + draw
  Napi::Value Render(const Napi::CallbackInfo& i) {
    auto o = i[0].As<Napi::Object>();
    gs_render_params p{};
    memcpy(p.proj, o.Get("proj").As<Napi::Float32Array>().Data(), 64);
    memcpy(p.modelview, o.Get("modelview").As<Napi::Float32Array>().Data(), 64);
    p.width = o.Get("width").As<Napi::Number>().Uint32Value();
    p.height = o.Get("height").As<Napi::Number>().Uint32Value();
    p.focal = o.Get("focal").As<Napi::Number>().FloatValue();
    if (o.Has("cutout")) { p.has_cutout = 1; memcpy(p.cutout16, o.Get("cutout").As<Napi::Float32Array>().Data(), 64); }
    if (o.Has("depth")) p.depth_in = o.Get("depth").As<Napi::Float32Array>().Data();  // gl.readPixels(DEPTH) of the scene so far
    p.out_format = GS_FORMAT_RGBA8;
    p.flags = Blend8(o);
    Check(i.Env(), gs_render(ctx_, &p, i[1].As<Napi::Uint8Array>().Data(), nullptr));
    return i.Env().Undefined();
  }
  // renderScene({proj, width, height, focal, depth?: Float32Array, blendUnorm8?}, [{first, count, modelview, cutout?}, ...], Uint8Array color,
  //             Uint8Array out)  <- the draws of every gaussian_splatting entity of the page, in DOM order (sortObjects false),
  // over the opaque pass: color = gl.readPixels(RGBA, UNSIGNED_BYTE) and depth = the window-space depth buffer read back
  // after the spheres and sky were drawn; each entity's {first, count} is its range of the shared table (filled by
  // insert / insertPly at the end of that range), modelview its getModelViewMatrix(camera), cutout its worldToCutout.
  Napi::Value RenderScene(const Napi::CallbackInfo& i) {
    auto o = i[0].As<Napi::Object>();
    gs_render_params p{};
    memcpy(p.proj, o.Get("proj").As<Napi::Float32Array>().Data(), 64);
    p.width = o.Get("width").As<Napi::Number>().Uint32Value();
    p.height = o.Get("height").As<Napi::Number>().Uint32Value();
    p.focal = o.Get("focal").As<Napi::Number>().FloatValue();
    if (o.Has("depth")) p.depth_in = o.Get("depth").As<Napi::Float32Array>().Data();
    p.out_format = GS_FORMAT_RGBA8;
    p.flags = Blend8(o);
    auto list = i[1].As<Napi::Array>();
    std::vector<gs_object> objs(list.Length());
    for (uint32_t k = 0; k < list.Length(); ++k) {
      auto e = list.Get(k).As<Napi::Object>();
      gs_object& g = objs[k];
      g = gs_object{};
      g.first = e.Get("first").As<Napi::Number>().Uint32Value();
      g.count = e.Get("count").As<Napi::Number>().Uint32Value();
      memcpy(g.modelview, e.Get("modelview").As<Napi::Float32Array>().Data(), 64);
      if (e.Has("cutout")) { g.has_cutout = 1; memcpy(g.cutout16, e.Get("cutout").As<Napi::Float32Array>().Data(), 64); }
    }
    const void* color = i[2].IsUndefined() ? nullptr : i[2].As<Napi::Uint8Array>().Data();
    Check(i.Env(), gs_render_scene(ctx_, &p, objs.data(), (uint32_t)objs.size(), color, i[3].As<Napi::Uint8Array>().Data(), nullptr));
    return i.Env().Undefined();
  }
  // pickScene({proj, width, height, focal, depth?: Float32Array}, [{first, count, modelview, cutout?}, ...], Uint32Array xy)
  //   -> {splat: Uint32Array, object: Int32Array, depth: Float32Array, alpha: Float32Array}   <- what a cursor, gaze or
  // controller ray meets on a splat entity (A-Frame's raycaster only sees each entity's dummy quad): for each (x, y) pixel of
  // xy (row 0 = bottom) of the frame renderScene draws with these arguments, the splat where the pixel turns half opaque
  // (splat 0xFFFFFFFF = GS_PICK_NONE and object -1 where none does), its entity's index in the list, its window depth and
  // the pixel's alpha.  At most GS_MAX_PICKS points per call; synchronous, like renderScene.
  Napi::Value PickScene(const Napi::CallbackInfo& i) {
    auto o = i[0].As<Napi::Object>();
    gs_render_params p{};
    memcpy(p.proj, o.Get("proj").As<Napi::Float32Array>().Data(), 64);
    p.width = o.Get("width").As<Napi::Number>().Uint32Value();
    p.height = o.Get("height").As<Napi::Number>().Uint32Value();
    p.focal = o.Get("focal").As<Napi::Number>().FloatValue();
    if (o.Has("depth")) p.depth_in = o.Get("depth").As<Napi::Float32Array>().Data();
    p.out_format = GS_FORMAT_RGBA8;
    auto list = i[1].As<Napi::Array>();
    std::vector<gs_object> objs(list.Length());
    for (uint32_t k = 0; k < list.Length(); ++k) {
      auto e = list.Get(k).As<Napi::Object>();
      gs_object& g = objs[k];
      g = gs_object{};
      g.first = e.Get("first").As<Napi::Number>().Uint32Value();
      g.count = e.Get("count").As<Napi::Number>().Uint32Value();
      memcpy(g.modelview, e.Get("modelview").As<Napi::Float32Array>().Data(), 64);
      if (e.Has("cutout")) { g.has_cutout = 1; memcpy(g.cutout16, e.Get("cutout").As<Napi::Float32Array>().Data(), 64); }
    }
    auto xy = i[2].As<Napi::Uint32Array>();
    const uint32_t n = (uint32_t)(xy.ElementLength() / 2);
    std::vector<gs_pick> hits(n ? n : 1);
    Napi::Env env = i.Env();
    Check(env, gs_pick_scene(ctx_, &p, objs.data(), (uint32_t)objs.size(), xy.Data(), n, hits.data()));
    if (env.IsExceptionPending()) return env.Undefined();
    auto splat = Napi::Uint32Array::New(env, n);
    auto object = Napi::Int32Array::New(env, n);
    auto depth = Napi::Float32Array::New(env, n);
    auto alpha = Napi::Float32Array::New(env, n);
    for (uint32_t k = 0; k < n; ++k) {
      splat[k] = hits[k].splat;
      object[k] = hits[k].object;
      depth[k] = hits[k].depth;
      alpha[k] = hits[k].alpha;
    }
    auto r = Napi::Object::New(env);
    r.Set("splat", splat);
    r.Set("object", object);
    r.Set("depth", depth);
    r.Set("alpha", alpha);
    return r;
  }
  // renderSceneXR([eyeL, eyeR] {proj, width, height, focal, x, y, blendUnorm8?}, [{first, count, modelview, cutout?,
  //                eyeModelviews: [Float32Array, Float32Array]}, ...], layer {color: Uint8Array, depth?: Float32Array, pitch,
  //                rows})  <- an XR frame of every entity of the page, drawn IN PLACE into the XR layer's one framebuffer:
  // each entity's tick() sort from the head camera (modelview = its getModelViewMatrix()), its draw once per eye with
  // eyeModelviews[e] = getModelViewMatrix(eyeCamera e) at that eye's viewport (x, y, width, height) = layer.getViewport(view
  // e); both eyes share one viewport size and the layer's one depth buffer.  One gs_render_scene_stereo_target: one sort,
  // both eyes in one pass, only the two eye rectangles read and written.
  Napi::Value RenderSceneXR(const Napi::CallbackInfo& i) {
    auto eyes_in = i[0].As<Napi::Array>();
    gs_render_params eyes[2] = {};
    uint32_t eye_xy[4];
    for (uint32_t e = 0; e < 2; ++e) {
      auto o = eyes_in.Get(e).As<Napi::Object>();
      memcpy(eyes[e].proj, o.Get("proj").As<Napi::Float32Array>().Data(), 64);
      eyes[e].width = o.Get("width").As<Napi::Number>().Uint32Value();
      eyes[e].height = o.Get("height").As<Napi::Number>().Uint32Value();
      eyes[e].focal = o.Get("focal").As<Napi::Number>().FloatValue();
      eyes[e].out_format = GS_FORMAT_RGBA8;
      eyes[e].flags = Blend8(o);
      eye_xy[2 * e] = o.Get("x").As<Napi::Number>().Uint32Value();
      eye_xy[2 * e + 1] = o.Get("y").As<Napi::Number>().Uint32Value();
    }
    auto list = i[1].As<Napi::Array>();
    const uint32_t n = list.Length();
    std::vector<gs_object> objs(n);
    std::vector<float> eye_mv(2 * (size_t)n * 16);
    for (uint32_t k = 0; k < n; ++k) {
      auto e = list.Get(k).As<Napi::Object>();
      gs_object& g = objs[k];
      g = gs_object{};
      g.first = e.Get("first").As<Napi::Number>().Uint32Value();
      g.count = e.Get("count").As<Napi::Number>().Uint32Value();
      memcpy(g.modelview, e.Get("modelview").As<Napi::Float32Array>().Data(), 64);
      if (e.Has("cutout")) { g.has_cutout = 1; memcpy(g.cutout16, e.Get("cutout").As<Napi::Float32Array>().Data(), 64); }
      auto mvs = e.Get("eyeModelviews").As<Napi::Array>();
      for (uint32_t s = 0; s < 2; ++s) memcpy(&eye_mv[((size_t)s * n + k) * 16], mvs.Get(s).As<Napi::Float32Array>().Data(), 64);
    }
    auto l = i[2].As<Napi::Object>();
    gs_target layer = {};
    layer.color = l.Get("color").As<Napi::Uint8Array>().Data();
    if (l.Has("depth")) layer.depth = l.Get("depth").As<Napi::Float32Array>().Data();
    layer.pitch = l.Get("pitch").As<Napi::Number>().Uint32Value();
    layer.rows = l.Get("rows").As<Napi::Number>().Uint32Value();
    Check(i.Env(), gs_render_scene_stereo_target(ctx_, eyes, objs.data(), eye_mv.data(), n, &layer, eye_xy, nullptr));
    return i.Env().Undefined();
  }
  gs_context* ctx_ = nullptr;
};
Napi::Object InitAll(Napi::Env env, Napi::Object exports) { return Splats::Init(env, exports); }
NODE_API_MODULE(gsplat_b200, InitAll)
