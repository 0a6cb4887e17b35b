/*
 * vmap_b200 -- C ABI of the H100-native (sm_90a) vMAP training-step library (libvmap_b200.so).
 *
 * The reference (kxhit/vMAP) is pure Python and has no FFI; its "operator interface"
 * for this path is the set of call sites in train.py.  Each entry point below replaces
 * the reference lines cited next to it.  Conventions:
 *   - plain C types only; every tensor argument is a DEVICE pointer owned by the caller
 *     (the library never frees, reallocates or keeps a caller pointer after return);
 *   - all work is enqueued on the cudaStream_t passed as `stream` (void* here so the
 *     header needs no CUDA include); nothing synchronises internally;
 *   - return 0 on success, a negative VMB_E_* code otherwise (vmb_last_error() has text);
 *     the reference's exit(-1) conditions (render_rays.py:88-90) become a device status
 *     word, never a process exit;
 *   - a handle is not thread safe; distinct handles are independent.
 *
 * Packed ensemble state ("param block"): one fp32 row per object, `vmb_param_stride()`
 * floats long, holding the 15 trainable tensors of one object in the order of
 * OccupancyMap.named_parameters() (model.py:17-52) followed by UniDirsEmbed.B_layer.weight
 * (embedding.py:75-76); offsets from vmb_param_offsets().  grads / Adam m / Adam v use
 * the same layout.
 */
#ifndef VMAP_B200_H
#define VMAP_B200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vmb_handle vmb_handle;

enum {
  VMB_OK = 0,
  VMB_E_ARG = -1,       /* bad argument / unsupported shape            */
  VMB_E_CUDA = -2,      /* CUDA runtime error (see vmb_last_error)     */
  VMB_E_NOMEM = -3,
  VMB_E_UNSUPPORTED = -4
};

/* vmb_step_args.impl */
enum {
  VMB_IMPL_AUTO = 0,
  VMB_IMPL_FP32 = 1,    /* CUDA-core fp32 kernel, any hidden size (parity anchor)            */
  VMB_IMPL_UMMA = 2,    /* wgmma fp16-operand fused kernel, hidden = 32 (the fast path): counts, step,
                           gradient reduction and (with fuse_adam) AdamW in ONE launch, n_samples <= 32        */
  VMB_IMPL_LAYERWISE = 3 /* wgmma GEMM per layer over all points, hidden = 64/128/256 (bg / iMAP) */
};

/* status word bits (vmb_step_args.status / vmb_adam_args.status, device int[4]) */
enum {
  VMB_ST_LOSS_EXPLODE = 1,   /* some per-object loss term > 1e5  (render_rays.py:88-90)      */
  VMB_ST_NONFINITE = 2       /* non-finite loss                                               */
};

#define VMB_N_TENSORS 15

/* ---- layout queries (host only, no GPU needed) --------------------------------------- */
/* number of trainable floats per object: 4H^2 + 225H + 4 + 63 for n_freq = 6             */
int vmb_param_count(int hidden, int n_freq);
/* row pitch of the param block in floats (param_count rounded up to 32)                   */
int vmb_param_stride(int hidden, int n_freq);
/* fills offsets[15] / sizes[15] (floats) in named_parameters() order, PE last             */
int vmb_param_offsets(int hidden, int n_freq, int* offsets, int* sizes);
/* bytes per object of the fp16 tensor-core weight image written by vmb_adam (0 if the
 * UMMA path does not support this hidden size)                                            */
int vmb_image_bytes(int hidden, int n_freq);
const char* vmb_version(void);

/* ---- lifetime ------------------------------------------------------------------------ */
/* Allocates per-handle scratch only (mask counts etc.).  Replaces nothing in the
 * reference; it is the moral equivalent of `optimiser = torch.optim.AdamW(...)`
 * (train.py:67) + `update_vmap` (utils.py:30-34) creating the stacked state.             */
int vmb_create(vmb_handle** out, int device, int max_obj, int hidden, int n_freq);
void vmb_destroy(vmb_handle* h);
const char* vmb_last_error(const vmb_handle* h);

/* ---- K0+K1: fused forward + loss + backward ------------------------------------------ */
/* One optimisation step's forward/backward for a stack of objects.  Replaces
 *   vmap(pe_model)(...), vmap(fc_model)(...)        train.py:293-294  (embedding.py:82-91, model.py:54-85)
 *   loss.step_batch_loss(...)                       train.py:303-306  (loss.py:5-62, render_rays.py:4-96)
 *   batch_loss.backward()                           train.py:324
 * `*_stride` = elements between consecutive objects, so that the per-iteration slices of
 * train.py:271-277 can be passed without a copy.                                          */
typedef struct vmb_step_args {
  int n_obj, n_rays, n_samples;     /* B, R, S                                             */
  int impl;                         /* VMB_IMPL_*                                          */
  const float* pcs;          long long pcs_stride;        /* [B][R][S][3] sample points    */
  const float* z_vals;       long long z_stride;          /* [B][R][S]                     */
  const float* gt_depth;     long long gt_depth_stride;   /* [B][R]                        */
  const float* gt_colour;    long long gt_colour_stride;  /* [B][R][3]  (rgb/255)          */
  const unsigned char* sem;  long long sem_stride;        /* [B][R] 0 other,1 this,2 unknown */
  const unsigned char* mask_depth; long long mask_stride; /* [B][R] bool valid depth       */
  const float* params;              /* [B][stride] fp32 master weights                     */
  const void*  image;               /* [B][image_bytes] fp16 weight image (UMMA path) or 0 */
  const float* scale;               /* [B] obj_scale buffer (embedding.py:80)              */
  float* grads;                     /* [B][stride], ACCUMULATED into (zero on entry; vmb_adam re-zeroes); unused with fuse_adam on hidden 32 */
  float* loss_terms;                /* [B][4] L_depth, L_colour, L_opacity, weighted total (overwritten) */
  float* r_depth;                   /* optional [B][R]      rendered depth                 */
  float* r_var;                     /* optional [B][R]      rendered variance              */
  float* r_colour;                  /* optional [B][R][3]                                  */
  float* r_opacity;                 /* optional [B][R]                                     */
  const int* counts;                /* optional [B][4] mask counts N_d,N_o,N_s,0 from
                                       vmb_mask_counts (+ all-reduce for ray-sharded iMAP);
                                       NULL = computed internally                          */
  float colour_scaling;             /* 5.0  (loss.py:6)                                    */
  float opacity_scaling;            /* 10.0 (loss.py:6)                                    */
  int   backward;                   /* 1 = forward+backward, 0 = forward/loss only         */
  int   fuse_adam;                  /* 1 = also do vmb_adam's work for this stack (optimiser.step(); zero_grad(),
                                       train.py:325-326) in the same call: hidden 32 runs it inside the step kernel
                                       (the last CTA to finish an object reduces that object's gradient partials in a
                                       fixed order and applies AdamW -- `grads` is then neither read nor written);
                                       other hidden sizes launch the AdamW kernel behind the step.  `params` and `image`
                                       are updated in place.  Needs backward = 1 and the fields below.               */
  void* k1_start_event;             /* optional cudaEvent_t recorded right before / after   */
  void* k1_stop_event;              /*   the fused K1 launch (roofline timing in bench.py)  */
  /* ---- only read when fuse_adam = 1 (same meaning as in vmb_adam_args) ---------------- */
  float* exp_avg;                   /* [B][stride] in/out                                   */
  float* exp_avg_sq;                /* [B][stride] in/out                                   */
  int*   step_counter;              /* optional DEVICE int[n_obj]: per-object step numbers  */
  int    step;                      /* 1-based step number when step_counter == NULL        */
  float  lr, beta1, beta2, eps, weight_decay;
  int    guard_loss;                /* 1 = skip an object's update and raise the status bits if its loss explodes */
  int*   status;                    /* optional device int[4], bits OR-ed in                */
  float* loss_sum;                  /* optional device float: receives the step's scalar loss, sum over objects of the
                                       weighted totals (`loss.sum()` of loss.py:59-62), so the caller needs no reduction
                                       launch of its own                                     */
} vmb_step_args;

int vmb_step(vmb_handle* h, const vmb_step_args* a, void* stream);

/* Mask counts only (the normalisers of render_rays.py:68,86): out[B][4] int.
 * Exposed separately so that a ray-sharded run can all-reduce them before vmb_step.       */
int vmb_mask_counts(vmb_handle* h, int n_obj, int n_rays,
                    const unsigned char* sem, long long sem_stride,
                    const unsigned char* mask_depth, long long mask_stride,
                    int* out_counts, void* stream);

/* ---- K2: fused stacked AdamW --------------------------------------------------------- */
/* Replaces optimiser.step(); optimiser.zero_grad(set_to_none=True) (train.py:325-326)
 * for the stacked leaves registered by update_vmap (utils.py:33): torch.optim.AdamW with
 * decoupled weight decay on every tensor (biases and PE directions included).             */
typedef struct vmb_adam_args {
  int n_obj;
  int step;                 /* 1-based step number t used for bias correction             */
  float* params;            /* [B][stride] in/out                                         */
  float* grads;             /* [B][stride] in; zeroed on exit if zero_grads               */
  float* exp_avg;           /* [B][stride] in/out                                         */
  float* exp_avg_sq;        /* [B][stride] in/out                                         */
  void*  image;             /* optional [B][image_bytes]: refreshed fp16 weight image     */
  const float* loss_terms;  /* optional [B][4]: update is skipped and VMB_ST_LOSS_EXPLODE
                               raised if any term > 1e5 or non-finite                     */
  int*   status;            /* optional device int[4], bits OR-ed in                      */
  float lr, beta1, beta2, eps, weight_decay;
  int   zero_grads;
  int*  step_counter;       /* optional DEVICE int[n_obj]: when set, object b uses t = step_counter[b] + 1
                               instead of `step` and the kernel increments every counter, so that a captured
                               CUDA graph of the step can be replayed; per-object numbers let objects that
                               joined the stack later keep a correct bias correction (SURVEY.md 8(f)3)       */
  const float* grad_scale;  /* optional DEVICE float: gradients are multiplied by it on the way in (the upstream
                               gradient autograd hands to `loss.backward()`, train.py:324), so the caller needs no
                               scaling pass over `grads`                                                     */
} vmb_adam_args;

int vmb_adam(vmb_handle* h, const vmb_adam_args* a, void* stream);

/* (Re)build the fp16 weight image from the fp32 master weights (after init / checkpoint
 * load / update_vmap re-stacking).                                                        */
int vmb_build_image(vmb_handle* h, int n_obj, const float* params, void* image, void* stream);

/* ---- forward only -------------------------------------------------------------------- */
/* Replaces Trainer.eval_points' per-chunk pe()+fc_occ_map() (trainer.py:77-90), batched
 * over objects: points [B][N][3] -> alpha [B][N] (raw*10, model.py:77), colour [B][N][3]. */
typedef struct vmb_forward_args {
  int n_obj; long long n_points;
  const float* points; long long points_stride;   /* elements between objects              */
  const float* params; const float* scale;
  float* alpha;  long long alpha_stride;
  float* colour; long long colour_stride;
  const void* image;   /* optional fp16 weight image (vmb_image_bytes per object, kept current by vmb_adam /
                          vmb_build_image): hidden 32 then runs the forward half of the fused wgmma kernel,
                          hidden 64/128/256 the layer-wise wgmma GEMMs; NULL = fp32 CUDA-core kernel          */
} vmb_forward_args;

int vmb_forward(vmb_handle* h, const vmb_forward_args* a, void* stream);

/* ---- K3: batched depth-guided ray sampler -------------------------------------------- */
/* Replaces the per-object Python loop train.py:208-218 over
 * sceneObject.get_training_samples / sample_3d_points (vmap.py:319-459) and the
 * stack + /255 of train.py:255-260.  One launch for all objects.                          */
typedef struct vmb_sample_args {
  int n_obj;
  int n_frames, n_pix;              /* keyframe draws per object, pixels per draw          */
  int n_bins_cam2surface, n_bins;   /* n1, n2: S = n1 + n2                                 */
  int width, height;                /* keyframe images are stored [W][H] (vmap.py:137-141) */
  float min_bound, surface_eps, stop_eps;
  /* per-object keyframe buffers: arrays of B device pointers                              */
  const unsigned char* const* rgbs;     /* [KF][W][H][4] u8 (rgb + state)                  */
  const float* const* depths;           /* [KF][W][H]                                      */
  const float* const* t_wc;             /* [KF][4][4]                                      */
  const float* const* bbox;             /* [KF][4] u_lo,u_hi,v_lo,v_hi                     */
  const int* n_keyframes;               /* [B]                                             */
  const int* latest_kf;                 /* [B][2] last two keyframe slots                  */
  const float* rays_dir;                /* [W][H][3] cameraInfo.rays_dir_cache             */
  const float* bin_limits;              /* [3][33]: linspace(0,1,n+1) for n=n1+n2, n1, n2  */
  /* randomness: Philox4x32-10 keyed by (seed, object) unless injected arrays are given   */
  unsigned long long seed, offset;
  const long long* inj_kf;              /* optional [B][n_frames]                          */
  const float* inj_u_w; const float* inj_u_h;   /* optional [B][n_frames][n_pix]           */
  const float* inj_u_z;                 /* optional [B][N][S]                              */
  const float* inj_nrm;                 /* optional [B][N][n2]  (already scaled by eps/3)  */
  /* outputs, N = n_frames*n_pix rays per object                                           */
  float* pcs;                /* [B][N][S][3]                                               */
  float* z_vals;             /* [B][N][S]                                                  */
  float* gt_depth;           /* [B][N]                                                     */
  float* gt_colour;          /* [B][N][3]  rgb/255 (train.py:257)                          */
  unsigned char* gt_rgb_u8;  /* optional [B][N][3] raw bytes as the reference returns them */
  unsigned char* sem;        /* [B][N]                                                     */
  unsigned char* mask_depth; /* [B][N]                                                     */
  /* Shared keyframe store (SURVEY.md 8(f)2; optional).  When store_rgbx != NULL the per-object pointer
   * tables rgbs/depths/t_wc/bbox above are ignored: every frame is stored once (instead of once per
   * object, vmap.py:137-176) and the pixel state the reference keeps in rgbs_batch[...,3] is derived
   * from the instance image as train.py:126-128 builds it (id == obj -> 1, id == -1 -> 2, else 0).  */
  const unsigned char* store_rgbx;  /* [slots][W][H][4] u8: r,g,b,unused                           */
  const float* store_depth;         /* [slots][W][H]                                               */
  const int* store_inst;            /* [slots][W][H] instance id per pixel (-1 = unknown)          */
  const float* store_t_wc;          /* [slots][4][4]                                               */
  const int* kf_slot;               /* [B][kf_stride] store slot of each object's keyframe         */
  const float* kf_bbox;             /* [B][kf_stride][4] u_lo,u_hi,v_lo,v_hi                       */
  const int* obj_id;                /* [B] instance id of each object                              */
  int kf_stride;
  /* Optional device-resident draw counter: when set it replaces `offset`, so a captured CUDA graph of a whole
   * frame (sampler + its optimisation steps) draws fresh samples on every replay (the caller increments it). */
  const unsigned long long* offset_dev;
} vmb_sample_args;

int vmb_sample(vmb_handle* h, const vmb_sample_args* a, void* stream);

/* ---- K4: frame ingest ----------------------------------------------------------------------------
 * One GPU pass over the instance image of a new frame.  Replaces the per-frame numpy loop of
 * dataset.py:101-131 (np.unique, a boolean mask per instance, utils.get_bbox2d_batch utils.py:75-84,
 * utils.enlarge_bbox utils.py:36-57, the "inst[obj_ == 0] = 0" relabel) and, with the shared keyframe
 * store, the per-object state-mask build and full-frame copies of train.py:121-141.
 * Images are stored [W][H] as the reference keeps them (dataset.py:87-91 transposes).                */
typedef struct vmb_ingest_args {
  int width, height;
  const int* inst;               /* [W][H] int32 instance id per pixel; ids outside [0,max_id) are not tabulated */
  const int* cls;                /* optional [W][H] int32 semantic class per pixel                               */
  int max_id;
  float bbox_scale;              /* dataset bbox_scale (enlarge_bbox's scale)                                    */
  int min_extent;                /* instances with an extent <= this are dropped (dataset.py:119 uses 10)        */
  const unsigned char* bg_class; /* optional [n_class]: 1 = background class (dataset.py:106)                    */
  int n_class;
  int* stats;                    /* out [max_id][8]: count, u_min, u_max+1, v_min, v_max+1, cls_min, cls_max, keep */
  float* bbox;                   /* out [max_id][4]: enlarged u_lo,u_hi,v_lo,v_hi (meaningful where keep)        */
  /* optional fused write of the frame into a slot of the shared keyframe store (all or none of dst_*)           */
  const unsigned char* rgb;      /* [W][H][3] u8                                                                 */
  const float* depth;            /* [W][H]                                                                       */
  unsigned char* dst_rgbx;       /* [W][H][4]                                                                    */
  float* dst_depth;              /* [W][H]                                                                       */
  int* dst_inst;                 /* [W][H]: dropped instances relabelled 0 (dataset.py:128), -1 kept             */
} vmb_ingest_args;

int vmb_ingest_frame(vmb_handle* h, const vmb_ingest_args* a, void* stream);

/* ---- K5: meshing -----------------------------------------------------------------------------------
 * Marching cubes on a dense fp32 volume.  Replaces skimage.measure.marching_cubes and the trimesh transforms of
 * Trainer.meshing (trainer.py:53-64, vis.py:6-19).  Volume [nx][ny][nz] (z fastest, nx, ny, nz >= 2); a corner is
 * inside when v > level; one vertex per crossed grid edge at a + t (b - a), t = (level - v_a) / (v_b - v_a), a the
 * lower-index end; vertex normal = the negated central-difference gradient (one-sided at the border) interpolated
 * along the edge, mapped by the inverse transpose of `affine` and normalised.  Triangles wind so that their
 * right-hand normal points from inside to outside (after `affine`, when its determinant is positive).  Order:
 * vertices by (grid-point linear index, edge axis x < y < z), faces by (cell linear index, case-table order).
 * Two calls with ONE host sync between them:
 *   vmb_mc_count  classifies the volume and writes the totals {vertices, faces} to totals[2];
 *   vmb_mc_emit   writes vertices / normals / faces of the volume given to the last vmb_mc_count on this handle
 *                 (same pointer and shape; VMB_E_ARG otherwise) into buffers sized from those totals.
 * An empty result (no crossing) is a success with zero totals.                                          */
typedef struct vmb_mc_args {
  const float* volume;           /* [nx][ny][nz]                                                                 */
  int nx, ny, nz;
  float level;                   /* 0.5 in Trainer.meshing (vis.py:6)                                             */
  float affine[12];              /* row-major 3x4 index -> world map (x_w = A[:, :3] x_i + A[:, 3]); host values   */
  int* totals;                   /* count: out device int[2] = number of vertices, faces                          */
  float* vertices;               /* emit: out [V][3]                                                              */
  float* normals;                /* emit: optional out [V][3]                                                     */
  int* faces;                    /* emit: out [F][3] vertex indices                                               */
  long long max_vertices, max_faces;   /* emit: capacities of the buffers above (entries beyond are not written) */
} vmb_mc_args;

int vmb_mc_count(vmb_handle* h, const vmb_mc_args* a, void* stream);
int vmb_mc_emit(vmb_handle* h, const vmb_mc_args* a, void* stream);

/* Object-pixel unprojection.  Replaces the open3d point cloud of sceneObject.get_bound (vmap.py:270-286): every
 * pixel of the object's first n_keyframes keyframes that belongs to the object and has depth > 0 becomes the world
 * point t_wc . [(u-cx) z/fx, (v-cy) z/fy, z, 1] (u indexes W, v indexes H, as cameraInfo), compacted in
 * (keyframe, u, v) order.  Per-object buffers: belongs = state byte rgbs[kf][u][v][3] == 1.  Shared keyframe store
 * (store_depth != NULL): belongs = store_inst[kf_slot[kf]][u][v] == obj_id.  `count` always receives the number of
 * selected pixels; `points` (optional) receives the first min(count, max_points) of them, so a caller that does
 * not know the count calls once without `points`, syncs, and calls again.                                      */
typedef struct vmb_unproject_args {
  int width, height, n_keyframes;
  float fx, fy, cx, cy;
  const unsigned char* rgbs;     /* per-object: [KF][W][H][4] u8, state in byte 3                                 */
  const float* depths;           /* per-object: [KF][W][H]                                                        */
  const float* t_wc;             /* per-object: [KF][4][4]                                                        */
  const float* store_depth;      /* store: [slots][W][H]                                                          */
  const int* store_inst;         /* store: [slots][W][H]                                                          */
  const float* store_t_wc;       /* store: [slots][4][4]                                                          */
  const int* kf_slot;            /* store: [n_keyframes] slot of each keyframe                                    */
  int obj_id;                    /* store: instance id of the object                                              */
  int* count;                    /* out device int                                                                */
  float* points;                 /* optional out [max_points][3]                                                  */
  long long max_points;
} vmb_unproject_args;

int vmb_unproject(vmb_handle* h, const vmb_unproject_args* a, void* stream);

/* ---- K6: 3-D reconstruction metrics ----------------------------------------------------------------
 * The arithmetic under metric/eval_3D_obj.py and eval_3D_scene.py: box crop, area-weighted surface sampling and exact
 * nearest-neighbour distances.  Means and ratios over the distances are left to the caller.
 *
 * Box crop (trimesh slice_plane with the six faces of an oriented box): each face of an indexed mesh is clipped
 * against the box's half-spaces (Sutherland-Hodgman in fp64, fp32 out, at most 9 vertices) and fan-triangulated from the first
 * clipped vertex.  Output: a triangle soup [T][3][3] ordered by (input face, fan order).  Faces wholly inside are
 * copied unchanged, faces wholly outside (or with an index outside [0, n_vertices)) give nothing.
 * Two calls with ONE host sync between them, as marching cubes:
 *   vmb_clip_count  writes T to *count (device int);
 *   vmb_clip_emit   writes the soup of the mesh and box given to the last vmb_clip_count on this handle (same
 *                   pointers, sizes and box; VMB_E_ARG otherwise) into a buffer sized from T.                 */
typedef struct vmb_clip_args {
  const float* vertices;         /* [V][3]                                                                       */
  long long n_vertices;
  const int* faces;              /* [F][3]                                                                       */
  long long n_faces;
  float center[3];               /* box center                                                                   */
  float rotation[9];             /* row-major 3x3 with the box axes as columns                                   */
  float extent[3];               /* full edge lengths along the three axes                                       */
  int* count;                    /* count: out device int = T                                                    */
  float* triangles;              /* emit: out [max_triangles][3][3]                                              */
  long long max_triangles;
} vmb_clip_args;

int vmb_clip_count(vmb_handle* h, const vmb_clip_args* a, void* stream);
int vmb_clip_emit(vmb_handle* h, const vmb_clip_args* a, void* stream);

/* Surface sampling (trimesh.sample.sample_surface): face areas 0.5 |e1 x e2| and their inclusive prefix in fp64; per
 * point face = searchsorted(prefix, u0 * total, side='left'), r = (u1, u2), r = |r - 1| when u1 + u2 > 1,
 * p = v0 + (r1 (v1 - v0) + r2 (v2 - v0)).  Randoms: Philox4x32-10 keyed by (seed, point index), or `uniforms`.
 * Syncs the stream once (to check the total area): a mesh of total area 0, or a face index outside [0, V), is
 * VMB_E_ARG.  n_points == 0 is a no-op.                                                                     */
typedef struct vmb_surface_sample_args {
  const float* vertices;         /* [V][3]                                                                       */
  long long n_vertices;
  const int* faces;              /* [F][3]                                                                       */
  long long n_faces;
  long long n_points;
  unsigned long long seed;
  const double* uniforms;        /* optional [n_points][3] (u0, u1, u2) in [0, 1): replaces Philox               */
  float* points;                 /* out [n_points][3]                                                            */
  int* face_index;               /* optional out [n_points]                                                      */
} vmb_surface_sample_args;

int vmb_surface_sample(vmb_handle* h, const vmb_surface_sample_args* a, void* stream);

/* Exact nearest neighbour: dist[i] = min_j |query_i - ref_j| (fp32 coordinates), index[i] = that j, ties to the lowest
 * j.  Uniform grid over ref's bounding box in handle scratch, shell search per query; no host sync.
 * n_ref == 0 is VMB_E_ARG; n_query == 0 is a no-op.                                                       */
typedef struct vmb_nn_args {
  const float* ref;              /* [n_ref][3]                                                                   */
  long long n_ref;
  const float* query;            /* [n_query][3]                                                                 */
  long long n_query;
  float* dist;                   /* out [n_query]                                                                */
  int* index;                    /* optional out [n_query]                                                       */
} vmb_nn_args;

int vmb_nn_dist(vmb_handle* h, const vmb_nn_args* a, void* stream);

/* ---- bring-up / test hook (not part of the reference-facing surface) --------------------------- */
/* Generic wgmma GEMM of the layer-wise wide-model path: D[M][N] = A[M][K1+K2] * B[N][K]^T, fp16 in,
 * fp32 accumulate.  a_mn/b_mn = 0: operand stored [rows][ld] with K contiguous; 1: stored [K][ld] with
 * M/N contiguous.  epi 0: out16 = relu(acc*scale + bias); 2: out32 (=|+=) acc*scale; 3: atomicAdd;
 * epi + 16 selects the weight-stationary kernel (a_mn = 0, N <= 256).                                */
int vmb_debug_gemm(int a_mn, int b_mn, int epi, int M, int N, int K1, int K2, const void* a1, long long a1_ld,
                   const void* a2, long long a2_ld, const void* b, long long b_ld, const float* bias, void* out16,
                   int ldo, float* out32, int ld32, int accumulate, int ksplit, float scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VMAP_B200_H */
