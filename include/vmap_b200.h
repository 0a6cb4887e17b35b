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
 * (train.py:67) + `update_vmap` (utils.py:30-34) creating the stacked state.
 * Scratch rule: every scratch buffer on the handle grows on demand, sized by the calls
 * that use it, and is freed by vmb_destroy.  A buffer is never moved once a CUDA graph
 * captured on a stream holds it (and never grows during a capture), so after a capture a
 * call that needs it larger fails with VMB_E_CUDA ("operation not permitted when stream
 * is capturing"): run the largest shape eagerly before capturing.                        */
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

/* Profiling build of vmb_step's fused hidden-32 training step (n_samples 10, impl AUTO / UMMA): the same launch and
 * results, with one thread per warpgroup stamping clock64() at every phase boundary of each tile (and %globaltimer at
 * kernel entry, last segment, finish start and exit) into `trace`
 * (device, 2 * min(#SMs, 192) rows of VMB_TRACE_STRIDE unsigned 64-bit words, row = 2 * CTA + warpgroup; the row
 * layout is described at uf::TR_STRIDE in k_step_fused.cuh).  For tools/step_phase_time.py.                         */
#define VMB_TRACE_STRIDE (16 + 64 * 20)
int vmb_step_trace(vmb_handle* h, const vmb_step_args* a, unsigned long long* trace, long long trace_words, void* stream);

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
  /* outputs, N = n_frames*n_pix rays per object (N < 2^29, VMB_E_ARG otherwise)            */
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
  /* Optional, appended for bundle adjustment (csrc/k_ba.cuh); 0 / NULL leave every launch as it was.
   * camera_frame != 0: take every keyframe's pose as identity (store and per-object mode), so pcs holds camera-frame
   * points q = d_c * z.  kf_out: [B][n_frames] the keyframe index each draw used (latest-two rule and injected
   * keyframes included).                                                                                           */
  int camera_frame;
  int* kf_out;
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

/* ScanNet relabel of a stored frame: the association's output (K7, vmb_assoc_finalize) replaces what the ingest wrote.
 * One launch, no sync: dst_inst[p] = labels[p] (int32; -1 = unknown), and for every id i in [0, max_id) the ingest's
 * tables are rebuilt: stats[i] = 0 except keep = (i < assoc_max_id and assoc_bbox[i + 1][0] != 0), bbox[i] = that
 * label's box [u_lo, u_hi, v_lo, v_hi] as f32 where kept, 0 elsewhere.                                          */
typedef struct vmb_relabel_args {
  int width, height;
  const long long* labels;       /* [W][H] int64 labels of vmb_assoc_finalize                                    */
  const long long* assoc_bbox;   /* [assoc_max_id + 1][5] its per-label box table (row r = label r - 1)          */
  int assoc_max_id;              /* the association's max_id, 1 .. max_id                                        */
  int max_id;                    /* rows of stats / bbox                                                         */
  int* stats;                    /* out [max_id][8] as vmb_ingest_args.stats (only keep is set)                  */
  float* bbox;                   /* out [max_id][4] as vmb_ingest_args.bbox                                      */
  int* dst_inst;                 /* out [W][H] the store slot's instance image                                   */
} vmb_relabel_args;

int vmb_store_relabel(vmb_handle* h, const vmb_relabel_args* a, void* stream);

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

/* ---- K7: ScanNet instance association --------------------------------------------------------------
 * utils.box_filter (utils.py:112-208) and the per-label 2-D boxes of dataset.py:263-283 for one frame, in three calls
 * on one handle, in this order, with the same args (images, max_id, tracks):
 *   vmb_assoc_classify  per id: pixel count, class minimum (background when bg_class[min] is set), valid-depth points,
 *                       eroded pixels (a pixel survives iff every in-image pixel within Chebyshev distance 6 has its
 *                       id: cv2.erode(ones(5,5), iterations=3)), eroded points and, for tracked ids, points inside the
 *                       tracked box (inclusive open3d test); then box_filter's branch in stats[id][6]
 *                       (VMB_ASSOC_*).  Points are x = (u-cx) z/fx, y = (v-cy) z/fy, camera_pose . [x y z 1] in fp64
 *                       with no FMA contraction.  No sync.
 *   vmb_assoc_voxel     for every MERGE / NEW id: its previous cloud (pool, merged ids only) followed by the selected
 *                       points in row-major (v, u) order, voxel-downsampled in fp64 (min_bound = min - voxel / 2,
 *                       key = floor((p - min_bound) / voxel), mean summed in input order), emitted into cloud_out in
 *                       ascending (id, kx, ky, kz) order; stats[id][7] = the id's output count.  Syncs the stream
 *                       ONCE: a voxel key outside [0, 65536) is VMB_E_ARG.
 *   vmb_assoc_finalize  labels from final_label (VMB_ASSOC_FINAL_*; an id labelled after a merge gets -1 on its
 *                       valid-depth pixels outside the box), per-label pixel boxes for labels -1 .. max_id-1, enlarged
 *                       as enlarge_bbox on python ints (margin = int((0.5 * bbox_scale) * extent) in fp64, clipped to
 *                       W-1 / H-1); a label whose margin is 0 is relabelled 0.  No sync.                             */
enum { VMB_ASSOC_ZERO = 0, VMB_ASSOC_MERGE = 1, VMB_ASSOC_NEW = 2, VMB_ASSOC_NEG = 3 };
enum { VMB_ASSOC_FINAL_ZERO = 0, VMB_ASSOC_FINAL_ID = 1, VMB_ASSOC_FINAL_NEG = 2 };

typedef struct vmb_assoc_args {
  int width, height;
  const int* inst;               /* [W][H] id per pixel (instance + 1, dataset.py:247); ids outside [1, max_id) are ignored */
  const int* cls;                /* optional [W][H] semantic class                                               */
  const float* depth;            /* [W][H] metres, <= 0 = no point                                               */
  int max_id;                    /* 1 .. 65536                                                                   */
  const unsigned char* bg_class; /* optional [n_class]: 1 = background class (dataset.py:187)                    */
  int n_class;
  double fx, fy, cx, cy;
  double camera_pose[16];        /* row-major 4x4 camera -> world; host values                                   */
  int min_pixels;                /* new ids need this many eroded pixels (dataset.py:184 uses 1500)              */
  double voxel_size;             /* 0.01 (utils.py:112)                                                          */
  double bbox_scale;             /* 0.2 (dataset.py:188)                                                         */
  const double* boxes;           /* [max_id][16]: tracked flag, center[3], R[:,j] * extent[j] / 2 for j = 0..2,
                                    then the three squared half-axis lengths                                     */
  const double* pool;            /* [n_pool][3] previous clouds                                                  */
  const int* cloud_off;          /* [max_id] first pool row of each id's cloud                                   */
  const int* cloud_cnt;          /* [max_id] rows of each id's cloud (0 = none)                                  */
  long long n_pool;
  int* stats;                    /* out [max_id][8]: pixels, class min, points, eroded pixels, eroded points,
                                    inside points, branch (VMB_ASSOC_*), voxelised points                        */
  double* cloud_out;             /* voxel: out [max_cloud_out][3], max_cloud_out >= n_pool + W * H               */
  long long max_cloud_out;
  const int* final_label;        /* finalize: [max_id] VMB_ASSOC_FINAL_*                                          */
  long long* labels;             /* finalize: out [W][H]                                                         */
  long long* bbox;               /* finalize: out [max_id + 1][5] per label + 1: kept, u_lo, u_hi, v_lo, v_hi;
                                    row 1 (label 0) is always the full frame [0, W, 0, H]                         */
  int relabel;                   /* finalize: 1 = relabel labels whose box is None to 0 (dataset.py:269-270);
                                    0 = leave box_filter's labels as they are                                    */
} vmb_assoc_args;

int vmb_assoc_classify(vmb_handle* h, const vmb_assoc_args* a, void* stream);
int vmb_assoc_voxel(vmb_handle* h, const vmb_assoc_args* a, void* stream);
int vmb_assoc_finalize(vmb_handle* h, const vmb_assoc_args* a, void* stream);

/* ---- K8: convex hulls and minimum-volume boxes -----------------------------------------------------
 * vmb_hull      exact 3-D convex hull of n_sets point sets in one call.  Set s is the next set_size[s * size_stride]
 *               points of `points` (negative sizes count as 0; the sizes are read and scanned on the device, so
 *               stats[:, 7] of vmb_assoc_voxel feeds it directly).  A vertex is an extreme point: a point on a facet
 *               or an edge is not one, and of several copies of an extreme point only the lowest index is flagged.
 *               Every predicate is exact (fp64 orientation with a static error filter, expansion arithmetic when
 *               the filter cannot decide).  status[s]: VMB_HULL_OK, TOO_FEW (fewer than 4 points), FLAT (all points
 *               coplanar, collinear or identical), BAD (the set reaches past n_points); a set that is not OK has no
 *               vertices and no facets.  Facets of set s are the rows 2 * (first point of s) + [0, facet_count[s]) of
 *               `facets`: point-index triples (a, b, c) with the outward normal along (b - a) x (c - a), a
 *               triangulation of the hull's boundary (its corners may include points that lie on a hull edge or
 *               inside a flat face).  facet_nbr[row][j] is the facet (relative to the set's first row) across the edge
 *               (v_j, v_j+1).  Vertices are compacted in (set, input order); vertex_offset[s] is set s's first
 *               entry and vertex_offset[n_sets] the total.  No host sync.                                     */
enum { VMB_HULL_OK = 0, VMB_HULL_TOO_FEW = 1, VMB_HULL_FLAT = 2, VMB_HULL_BAD = 3 };

typedef struct vmb_hull_args {
  const double* points;          /* [n_points][3], finite                                                         */
  long long n_points;
  const int* set_size;           /* device: size of set s at set_size[s * size_stride]                            */
  int size_stride;               /* >= 1 (ints)                                                                   */
  int n_sets;                    /* >= 1                                                                          */
  unsigned char* is_vertex;      /* out [n_points] 1 = extreme point of its set                                   */
  int* vertex_count;             /* out [n_sets]                                                                  */
  int* vertex_offset;            /* optional out [n_sets + 1]; required with vertices                             */
  int* vertices;                 /* optional out [n_points] extreme point indices, (set, input order)             */
  int* status;                   /* out [n_sets] VMB_HULL_*                                                       */
  int* facets;                   /* out [2 * n_points][3]                                                         */
  int* facet_nbr;                /* optional out [2 * n_points][3]                                                */
  int* facet_count;              /* out [n_sets]                                                                  */
} vmb_hull_args;

int vmb_hull(vmb_handle* h, const vmb_hull_args* a, void* stream);

/* vmb_obb_minvol  minimum-volume oriented box of one set from its hull (trimesh.bounds.oriented_bounds as
 *               vmap_b200/mesh.py restates it): for every distinct facet normal (unit, rounded to 1e-10) the height
 *               along it and the minimum-area rectangle of the projected hull vertices over the projected silhouette
 *               edge directions; the least volume wins, exact ties to the lexicographically smallest normal.  Pass
 *               the set's rows of vmb_hull's facets / facet_nbr, its vertices, and device pointers to its counts and
 *               status.  box = center[3], R[3][3] row-major (columns are the box axes, det +1), extent[3], fp64.
 *               box_status = VMB_HULL_OK or the hull's status.  No host sync.                                    */
typedef struct vmb_obb_args {
  const double* points;          /* the points vmb_hull was given                                                 */
  const int* facets;             /* [facet_count][3]                                                              */
  const int* facet_nbr;          /* [facet_count][3]                                                              */
  const int* facet_count;        /* device [1]                                                                    */
  const int* vertices;           /* [vertex_count] extreme point indices                                          */
  const int* vertex_count;       /* device [1]                                                                    */
  const int* status;             /* device [1] the set's VMB_HULL_* status                                        */
  long long max_facets;          /* upper bound of facet_count (sizes the scratch)                                */
  double* box;                   /* out [15]                                                                      */
  int* box_status;               /* out [1]                                                                       */
} vmb_obb_args;

int vmb_obb_minvol(vmb_handle* h, const vmb_obb_args* a, void* stream);

/* ---- K9: view rendering of the object map (vmap_b200/render.py; the rule is in csrc/k_render.cuh) ---------------
 * Rays [ray0, ray0 + n_rays) of a width x height camera (pixel (u, v) = ray u*height + v) are culled against up to
 * 1024 oriented boxes, sampled inside each hit box and composited front to back.  Per pass (0 coarse, 1 fine):
 *   vmb_render_count      pass 0 writes the hit table (nearest 16 hits per ray by (t0, source)), hit counts and the
 *                         overflow count; both passes write src_total, the samples of the pass per source.  Pass 1
 *                         reads zstar.  The caller reads src_total (one host sync) to size the emit buffers.
 *   vmb_render_emit       writes the pass's samples source-major (source, ray, k): points [sum][3] (world point minus
 *                         the source's offset, fp32), z [sum], and base[ray][hit], the first sample of each entry.
 *                         Must follow a count with the same arguments (VMB_E_ARG otherwise).
 *   (the caller runs vmb_forward per source on its contiguous segment: alpha [sum], colour [sum][3])
 *   vmb_render_composite  pass 0 writes zstar (-1 = none) and surf (merged index of the surface sample, -1 = none),
 *                         and the images when n_fine == 0; pass 1 composites coarse + fine into the images.
 * Images are full-view [width * height] device arrays; each call writes its rays only.  VMB_E_ARG on: width or
 * height <= 0, n_src outside [1, 1024], n_coarse < 1, n_fine < 0, fx or fy == 0, a non-finite pose / intrinsic /
 * box, a half-extent <= 0, near < 0 or far <= near.                                                                */
typedef struct vmb_render_args {
  int width, height;
  double fx, fy, cx, cy;
  double t_wc[12];               /* camera-to-world rows 0..2 of the 4x4, row-major; host values                   */
  double near_depth, far_depth;  /* cfg.min_depth, cfg.max_depth                                                   */
  double surface_eps;            /* fine band half-width (cfg.surface_eps)                                         */
  int n_src;                     /* 1..1024                                                                        */
  const double* boxes;           /* HOST [n_src][18]: center[3], R[3][3] row-major (columns = axes), half[3], offset[3] */
  const int* obj_id;             /* HOST [n_src] instance id written for a source's surface                       */
  long long ray0;
  int n_rays;
  int n_coarse, n_fine;          /* samples per hit box; per fine band (0 = coarse only)                           */
  int pass;                      /* 0 coarse, 1 fine                                                               */
  int* hit_src;                  /* [n_rays][16] source index, -1 past hit_count                                   */
  double* hit_t;                 /* [n_rays][16][2] (t0, t1)                                                       */
  int* hit_count;                /* [n_rays]                                                                       */
  int* overflow;                 /* count pass 0: out [1] rays with more than 16 hits                             */
  int* src_total;                /* count: out [n_src] samples of this pass per source                            */
  float* zstar;                  /* [n_rays] surface depth of the coarse composite, -1 = none                     */
  int* surf;                     /* [n_rays] merged index of the coarse surface sample, -1 = none                 */
  float* points;                 /* emit: out [sum][3]                                                             */
  float* z;                      /* emit: out [sum]                                                                */
  int* base;                     /* emit: out [n_rays][16]                                                         */
  const float* z_coarse;         /* composite: the coarse pass's z, alpha [sum], colour [sum][3], base             */
  const float* alpha_coarse;
  const float* colour_coarse;
  const int* base_coarse;
  const float* z_fine;           /* composite pass 1: the same for the fine pass                                   */
  const float* alpha_fine;
  const float* colour_fine;
  const int* base_fine;
  float* depth;                  /* out [width * height]                                                           */
  float* colour;                 /* out [width * height][3]                                                        */
  float* opacity;                /* out [width * height]                                                           */
  int* instance;                 /* out [width * height] obj_id of the surface source, -1 = none                   */
} vmb_render_args;

int vmb_render_count(vmb_handle* h, const vmb_render_args* a, void* stream);
int vmb_render_emit(vmb_handle* h, const vmb_render_args* a, void* stream);
int vmb_render_composite(vmb_handle* h, const vmb_render_args* a, void* stream);

/* ---- K10: camera tracking against the object map (vmap_b200/track.py; the rule is in csrc/k_track.cuh) -----------
 * Adds what neither code base has: the pose of a new RGB-D frame estimated against the map.  The reference reads GT
 * poses (dataset.py:135) or takes them from an external tracker in live mode (next_live_data); its unused
 * optimizer.args.pose_lr is the rate here.  Per iteration of a frame:
 *   vmb_track_step    once per group (one ensemble; hidden 32/64/128/256, same tiles and limits as the fp32 step):
 *                     per-slice mask counts, forward, render, loss and the backward to the sample points, reduced into
 *                     per-CTA fp64 partials of the 6-DoF pose gradient and the loss terms.  Reads the pose from `pose`
 *                     and each object's weights from params row rows[b] (a subset of a packed stack, no repacking).
 *   vmb_track_update  one small launch: sums every group's partials in a fixed order, runs Adam on the tangent and
 *                     applies Exp; writes the pose, the iteration's scalar loss and the per-object loss terms.
 * Everything stays on the device (no host sync), so a whole tracking loop can be captured as one CUDA graph.
 * VMB_E_ARG: bad counts, hidden != the handle's, missing pointers, partials too small, n_iter < 1, iter outside
 * [1, n_iter], bad rates; VMB_E_UNSUPPORTED: n_samples above the tile of the hidden size.  rows[] and the pose live on
 * the device: a row outside [0, n_rows) contributes nothing and sets VMB_TRACK_ST_BAD_ROW, a non-finite pose, loss or
 * gradient skips the update and sets VMB_ST_NONFINITE in `status`.                                                     */
#define VMB_TRACK_MAX_GROUPS 8
#define VMB_TRACK_PART 10              /* doubles per partial row: dL/dphi[3], dL/drho[3], L_d, L_c, L_o, 0           */
enum { VMB_TRACK_ST_BAD_ROW = 4 };

typedef struct vmb_track_group {
  int hidden;                    /* the ensemble's hidden size (must match the handle of vmb_track_step)            */
  int n_obj;                     /* B tracked objects                                                               */
  int n_rows;                    /* rows of the packed stack `params` / `scale`                                    */
  const int* rows;               /* device [B] params row of each tracked object                                   */
  int n_rays, n_samples;         /* R rays of this iteration's slice, S samples per ray                             */
  const float* pcs;          long long pcs_stride;        /* [B][R][S][3] camera-frame points q (identity-pose samples) */
  const float* z_vals;       long long z_stride;          /* [B][R][S]                                              */
  const float* gt_depth;     long long gt_depth_stride;   /* [B][R]                                                 */
  const float* gt_colour;    long long gt_colour_stride;  /* [B][R][3]                                              */
  const unsigned char* sem;  long long sem_stride;        /* [B][R]                                                 */
  const unsigned char* mask_depth; long long mask_stride; /* [B][R]                                                 */
  const float* params;           /* [n_rows][stride] fp32 weights                                                   */
  const float* scale;            /* [n_rows] obj_scale                                                              */
  double* partials;              /* [B * vmb_track_tiles(hidden, R, S)][VMB_TRACK_PART] scratch                     */
  long long max_partials;        /* rows available in `partials`                                                    */
  float* loss_terms;             /* optional [B][4] L_depth, L_colour, L_opacity, weighted total (written by update) */
} vmb_track_group;

typedef struct vmb_track_args {
  int n_groups;                  /* 1 .. VMB_TRACK_MAX_GROUPS                                                       */
  vmb_track_group group[VMB_TRACK_MAX_GROUPS];
  int n_iter;                    /* iterations of the frame (>= 1)                                                  */
  int iter;                      /* this iteration, 1-based (Adam's bias correction; moments restart at 1)          */
  double* pose;                  /* device [4][4] fp64 T_wc, in/out                                                 */
  double* adam;                  /* device [12] Adam moments m[6], v[6] of the tangent (phi, rho)                   */
  double lr_rot, lr_trans;       /* cfg.pose_lr by default                                                          */
  double beta1, beta2, eps;      /* 0.9, 0.999, 1e-8                                                                */
  float colour_scaling;          /* 5.0  (loss.py:6)                                                                */
  float opacity_scaling;         /* 10.0 (loss.py:6)                                                                */
  double* loss;                  /* optional device [n_iter]: loss[iter-1] = the iteration's loss (before the update)*/
  double* pose_hist;             /* optional device [n_iter+1][4][4]: the pose before iteration 1 and after each    */
  double* grad_hist;             /* optional device [n_iter][6]: each iteration's gradient (phi, rho)               */
  int* status;                   /* optional device int[4], bits OR-ed in                                           */
} vmb_track_args;

/* tiles (partial rows) per object of vmb_track_step for this shape, or a negative VMB_E_* code (host only)           */
int vmb_track_tiles(int hidden, int n_rays, int n_samples);
int vmb_track_step(vmb_handle* h, const vmb_track_args* a, int group, void* stream);
int vmb_track_update(vmb_handle* h, const vmb_track_args* a, void* stream);

/* ---- K11: bundle adjustment of keyframe poses (vmap_b200/ba.py; the rule is in csrc/k_ba.cuh) ------------------
 * Pose-only passes against a frozen map, between mapping frames: every keyframe pose the objects' keyframe tables hold
 * is moved by the same loss the mapping frame minimises.  Per iteration of a pass:
 *   vmb_ba_step    once per group (one ensemble; hidden 32/64/128/256, S as vmb_track_step): K10's forward, render,
 *                  loss and backward to the sample points, with the pose of each ray read from the fp64 pose table at
 *                  the frame its draw used; writes one fp64 row per ray (VMB_TRACK_PART doubles, as K10's partials).
 *   vmb_ba_update  one small launch: sums the rows per (object, draw) and per window frame in a fixed order, runs one
 *                  Adam on the stacked tangents of the window and applies Exp to each window pose in the table; after
 *                  the last iteration writes each window pose in fp32 to the targets.
 * VMB_E_ARG: bad counts, hidden != the handle's, missing pointers, rows or scratch too small, n_rays not a multiple of
 * n_pix_draw, n_win outside [1, VMB_BA_MAX_WIN], iter outside [1, n_iter], bad rates.  On the device: a draw whose
 * keyframe index or frame id is outside its table contributes nothing and sets VMB_BA_ST_BAD_FRAME (as does a window
 * entry >= n_poses); a row outside [0, n_rows) sets VMB_TRACK_ST_BAD_ROW; a non-finite loss, gradient or window pose
 * skips the iteration's update and sets VMB_ST_NONFINITE.  Window entries must be distinct.                         */
#define VMB_BA_MAX_WIN 1024
enum { VMB_BA_ST_BAD_FRAME = 8 };

typedef struct vmb_ba_group {
  int hidden;                    /* the ensemble's hidden size (must match the handle of vmb_ba_step)               */
  int n_obj;                     /* B objects                                                                       */
  int n_rows;                    /* rows of the packed stack `params` / `scale`                                    */
  const int* rows;               /* device [B] params row of each object                                           */
  int n_rays, n_samples;         /* R rays of this iteration's slice, S samples per ray                             */
  const float* pcs;          long long pcs_stride;        /* [B][R][S][3] camera-frame points q                    */
  const float* z_vals;       long long z_stride;          /* [B][R][S]                                              */
  const float* gt_depth;     long long gt_depth_stride;   /* [B][R]                                                 */
  const float* gt_colour;    long long gt_colour_stride;  /* [B][R][3]                                              */
  const unsigned char* sem;  long long sem_stride;        /* [B][R]                                                 */
  const unsigned char* mask_depth; long long mask_stride; /* [B][R]                                                 */
  const float* params;           /* [n_rows][stride] fp32 weights                                                   */
  const float* scale;            /* [n_rows] obj_scale                                                              */
  int n_pix_draw;                /* rays per draw: ray r of the slice belongs to draw r / n_pix_draw                */
  const int* kf_draw;  long long kf_draw_stride;          /* [B][R / n_pix_draw] keyframe index of each draw        */
  const int* kf_frame; int kf_stride;                     /* [B][kf_stride] frame id of each keyframe index (-1: none) */
  double* ray_rows;              /* [B][R][VMB_TRACK_PART] scratch: dL/dphi[3], dL/drho[3], L_d, L_c, L_o, 0       */
  long long max_ray_rows;        /* rows available in `ray_rows`                                                    */
} vmb_ba_group;

typedef struct vmb_ba_target {
  const int* frame_of;           /* device [n] frame id held by each entry (-1: none)                               */
  float* t_wc;                   /* device [n][4][4] fp32 poses to refresh (NULL: no target)                        */
  int n;
} vmb_ba_target;

typedef struct vmb_ba_args {
  int n_groups;                  /* 1 .. VMB_TRACK_MAX_GROUPS                                                       */
  vmb_ba_group group[VMB_TRACK_MAX_GROUPS];
  int n_iter;                    /* iterations of the pass (>= 1)                                                   */
  int iter;                      /* this iteration, 1-based (Adam's bias correction; moments restart at 1)          */
  double* poses;                 /* device [n_poses][4][4] fp64 pose table T_wc, in/out                             */
  int n_poses;
  const int* window;             /* device [n_win] distinct frame ids the pass moves (-1: padding)                  */
  int n_win;
  int hold;                      /* a frame id that never moves (the anchor, 0), or -1                              */
  double* adam;                  /* device [n_win][12] Adam moments m[6], v[6] per window entry                     */
  double* scratch;               /* device, >= 8 * sum_groups(n_obj * n_rays / n_pix_draw) + 6 * n_win doubles      */
  long long scratch_len;
  double lr_rot, lr_trans;       /* cfg.pose_lr by default                                                          */
  double beta1, beta2, eps;      /* 0.9, 0.999, 1e-8                                                                */
  float colour_scaling;          /* 5.0  (loss.py:6)                                                                */
  float opacity_scaling;         /* 10.0 (loss.py:6)                                                                */
  double* loss;                  /* optional device [n_iter]: loss[iter-1] = the iteration's loss (before the update)*/
  double* pose_hist;             /* optional device [n_iter+1][n_win][4][4]: poses before iteration 1 and after each */
  double* grad_hist;             /* optional device [n_iter][n_win][6]: each iteration's gradient per window entry  */
  vmb_ba_target target[2];       /* written after iteration n_iter                                                  */
  int* status;                   /* optional device int[4], bits OR-ed in                                           */
} vmb_ba_args;

int vmb_ba_step(vmb_handle* h, const vmb_ba_args* a, int group, void* stream);
int vmb_ba_update(vmb_handle* h, const vmb_ba_args* a, void* stream);

/* ---- K10 / K11 on the layer-wise tensor-core path (the rule is in csrc/k_track_lw.cuh) ------------------------------
 * The same step as vmb_track_step / vmb_ba_step for the wide models (hidden 64/128/256, n_freq 6), with the network
 * on the wgmma GEMMs of the layer-wise training path, reading each object's weights from the ensemble's fp16 image
 * `image` ([n_rows][vmb_image_bytes], as the AdamW launch writes it; row rows[b] for object b, as params).  Writes the
 * same rows as vmb_track_step (K10's partials: vmb_track_tiles rows per object) and vmb_ba_step (one row per ray), so
 * vmb_track_update and vmb_ba_update run unchanged.  No floating-point atomics: bitwise reproducible.
 * Argument checks as vmb_track_step / vmb_ba_step; VMB_E_ARG also for a NULL image; VMB_E_UNSUPPORTED for hidden 32
 * (stays on vmb_track_step / vmb_ba_step) and n_samples > 32.  On the device, besides the bits of K10 / K11: a
 * loss-scaled gradient that reaches the fp16 clamp (+-60000) sets VMB_TRACK_ST_CLAMP and adds to status[1] a lower
 * bound on the number of clamped values (the colour-hidden gradient and the rank-1 alpha term; the saturating
 * packs of the dY4..dY1 GEMMs are not counted).                                                                                              */
enum { VMB_TRACK_ST_CLAMP = 16 };
int vmb_track_step_lw(vmb_handle* h, const vmb_track_args* a, int group, const void* image, void* stream);
int vmb_ba_step_lw(vmb_handle* h, const vmb_ba_args* a, int group, const void* image, void* stream);

/* ---- K10 / K11 at hidden 32 on the fused wgmma tile (the rule is in csrc/k_track_fused.cuh) -------------------------
 * The same step as vmb_track_step / vmb_ba_step for the hidden-32 object models (n_freq 6), with the network on the
 * tile of the fused training step: one launch per call covers every object of the group, each object reading its fp16
 * weight image row rows[b] of `image` ([n_rows][vmb_image_bytes], as the AdamW launch writes it).  The forward and the
 * input-gradient chain only (no weight gradients); render, loss and pose terms in fp64 as K10.  Writes the same rows as
 * vmb_track_step (K10's partials: vmb_track_tiles rows per object, the per-ray terms summed per K10 tile in ray order)
 * and vmb_ba_step (one row per ray), so vmb_track_update and vmb_ba_update run unchanged.  No floating-point atomics:
 * bitwise reproducible.  Argument checks as the _lw pair; VMB_E_ARG also for a NULL image and a partials or ray-rows
 * buffer that is too small; VMB_E_UNSUPPORTED for hidden != 32 or n_freq != 6 (hidden 64/128/256 take the _lw pair) and
 * n_samples > 32.  On the device, besides the bits of K10 / K11: a loss-scaled head gradient (LS d(raw alpha),
 * LS d(raw colour)) past the fp16 clamp (+-60000) sets VMB_TRACK_ST_CLAMP and adds to status[1] the number of such
 * values, a lower bound on the clamped values (the saturating packs of the d_hc .. d_fc1 epilogues are not counted). */
int vmb_track_step_fused(vmb_handle* h, const vmb_track_args* a, int group, const void* image, void* stream);
int vmb_ba_step_fused(vmb_handle* h, const vmb_ba_args* a, int group, const void* image, void* stream);

/* ---- relocalisation: the tracking loss of many candidate poses at once and their top K (vmap_b200/reloc.py; the rule
 * is in csrc/k_reloc.cuh) ---------------------------------------------------------------------------------------------
 *   vmb_reloc_score   hidden 32: for each hypothesis h of the device table hyps [n_hyp][4][4] (fp64 T_wc), K10's loss
 *                     of group `group` of `a` at T_h on the group's slice (its camera-frame points, targets and masks as
 *                     vmb_track_step reads them; the mask counts are counted once and shared by every hypothesis), from
 *                     the fused tile's forward on the fp16 image `image` (as vmb_track_step_fused), summed in K10's order
 *                     (rays within each vmb_track_tiles tile, tiles, then the objects by vmb_track_update's tree), ADDED
 *                     to scores[h] (device [n_hyp] fp64: zero it before the first group).  On one group scores[h] is, bit
 *                     for bit, the loss vmb_track_update reports for an iteration from T_h on the same slice.  terms:
 *                     optional device [n_hyp][n_obj][4] fp64 per-object L_depth, L_colour, L_opacity, weighted total.
 *                     Reads a's colour_scaling, opacity_scaling and status (not its pose, adam or iteration fields); the
 *                     group's partials are checked as vmb_track_step checks them and not written.
 *   vmb_reloc_select  the k smallest of the device scores [n] on the device: idx [k] (int) ascending by score, ties to
 *                     the lower index, a non-finite score after every finite one; poses (optional) [k][4][4] the
 *                     matching rows of hyps.  No host read.
 * VMB_E_ARG: as vmb_track_step_fused, n_hyp outside [1, VMB_RELOC_MAX_HYP], k outside [1, min(n, VMB_RELOC_MAX_K)],
 * a NULL image, hyps, scores or idx.  VMB_E_UNSUPPORTED: hidden != 32 or n_freq != 6, n_samples > 32.  On the device: a
 * row outside [0, n_rows) contributes 0 and sets VMB_TRACK_ST_BAD_ROW.  No floating-point atomics: bitwise reproducible,
 * and a hypothesis's score does not depend on n_hyp.  The per-ray scratch ([n_hyp][n_obj][n_rays][3] fp64 on the
 * handle) follows the scratch rule (vmb_create): after a capture, a call with a larger n_hyp * n_obj * n_rays fails
 * with VMB_E_CUDA.  Registers as in k_reloc.cuh. */
#define VMB_RELOC_MAX_HYP 4096
#define VMB_RELOC_MAX_K 64
int vmb_reloc_score(vmb_handle* h, const vmb_track_args* a, int group, int n_hyp, const double* hyps, double* scores,
                    double* terms, const void* image, void* stream);
int vmb_reloc_select(vmb_handle* h, int n, const double* scores, const double* hyps, int k, int* idx, double* poses,
                     void* stream);

/* ---- joint map-and-pose step on the layer-wise path (iMAP: network weights and keyframe poses together; the rule is
 * in csrc/k_track_lw.cuh) ---------------------------------------------------------------------------------------------
 * One mapping iteration that also yields K11's per-ray pose rows, from ONE forward and backward:
 *   vmb_joint_step_lw  per object: world points p = R_f q + t_f (fp32 from an fp32 copy of the fp64 pose of the frame of
 *                      the ray's draw, as K11) from the camera-frame samples s->pcs, then vmb_step's layer-wise step on p
 *                      (mask counts, forward, render, loss, weight gradients accumulated into s->grads, loss_terms,
 *                      loss_sum and the optional rendered outputs), then the pose terms of every point from that step's
 *                      own embedding gradient and one row per ray into a->group[group].ray_rows (K11's layout; the loss
 *                      columns are 0: the iteration's loss is the mapping loss in loss_terms / loss_sum).
 * The caller then runs vmb_adam on the weights (the pose terms read the PE directions before it) and vmb_ba_update on
 * the same vmb_ba_args (one Adam + Exp over the window).  `s`: as vmb_step, with fuse_adam = 0, backward = 1, grads and
 * the fp16 image set, impl AUTO or LAYERWISE.  `a`: the pose table (poses, n_poses), status, and in group `group` the
 * draw layout, keyframe tables and ray rows of the same objects, rays and samples (its other fields are not read here).
 * pcs_world_out: optional [B][R][S][3] copy of the world points.  VMB_E_UNSUPPORTED for hidden 32; VMB_E_ARG as vmb_step
 * and vmb_ba_step, and for a group that does not match `s`.  On the device: a ray whose draw's frame is outside its table
 * is mapped at p = q, contributes nothing to the rows and sets VMB_BA_ST_BAD_FRAME.  No floating-point atomics on the
 * pose side: the rows are bitwise reproducible for a given embedding gradient.
 * Registers (ptxas -v, sm_90a), no spills: k_joint_world 32; k_tlw_pose and k_tlw_reduce as listed in k_track_lw.cuh. */
int vmb_joint_step_lw(vmb_handle* h, const vmb_step_args* s, const vmb_ba_args* a, int group, float* pcs_world_out,
                      void* stream);

/* ---- joint map-and-pose step on the fused hidden-32 step (vMAP: the objects' weights and keyframe poses together; the
 * rule is in csrc/k_step_fused.cuh and csrc/k_track_lw.cuh) ------------------------------------------------------------
 *   vmb_joint_step_fused  world points of all B objects in one launch (k_joint_world, as vmb_joint_step_lw), then vmb_step's
 *                      fused hidden-32 step on them (mask counts, forward, render, loss, backward, the ordered gradient
 *                      reduction and, with fuse_adam = 1, AdamW), whose PE backward also forms every point's dL/dt from
 *                      the pre-update directions, then one row per ray into a->group[group].ray_rows (K11's layout, loss
 *                      columns 0).  The caller then runs vmb_ba_update.
 * `s`: as vmb_step at hidden 32, with the image, backward = 1, impl AUTO or UMMA, fuse_adam 0 (gradients added into
 * s->grads) or 1.  `a`, `group` and pcs_world_out as vmb_joint_step_lw.  VMB_E_UNSUPPORTED for hidden 64/128/256 (they
 * take vmb_joint_step_lw); VMB_E_ARG as vmb_joint_step_lw.  The rows are the gradient of the mapping loss, so its
 * whole-batch empty-mask rule applies (a term is off for every object when one object's count of it is 0).  No
 * floating-point atomics on the pose side: the rows are bitwise reproducible.
 * Registers (ptxas -v, sm_90a), no spills: k_joint_world 32, k_joint_rows 68; k_step_fused JOINT as listed in
 * k_step_fused.cuh. */
int vmb_joint_step_fused(vmb_handle* h, const vmb_step_args* s, const vmb_ba_args* a, int group, float* pcs_world_out,
                         void* stream);

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
