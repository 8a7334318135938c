/* libepid -- H100-native (sm_90a) EPID image-analysis hot path.  C-ABI boundary.
 *
 * The reference (jrkerns/pylinac v3.46.0) is pure Python and has NO FFI of its own: its numerical
 * work goes through numpy / scipy.ndimage / scipy.signal call sites inside pylinac/core/image.py,
 * pylinac/core/array_utils.py, pylinac/core/profile.py and the module-level analyze() methods.
 * Each entry point below replaces one of those call sites (cited as file:line of the reference);
 * pylinac_b200/_native.py is the ctypes binding a maintainer would add (see INTEGRATION.md).
 *
 * Conventions
 *  - plain C, no exceptions; every function returns an int32 status (EPID_OK == 0, negative = error).
 *  - images are row-major [row=y][col=x]; a "batch" is n equal-sized frames, contiguous.
 *  - host pointers are owned by the caller; device memory is owned by ctx / batch handles.
 *  - calls are synchronous unless stated otherwise (they return after the result is in host memory).
 *  - there is NO CPU fallback: without a CUDA device every compute entry point returns EPID_ERR_NO_DEVICE.
 */
#ifndef EPID_H
#define EPID_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ----------------------------------------------------------------------------------------- status */
enum {
    EPID_OK = 0,
    EPID_ERR_NO_DEVICE = -1,      /* no CUDA device / driver */
    EPID_ERR_CUDA = -2,           /* CUDA runtime error, see epid_last_error() */
    EPID_ERR_INVALID = -3,        /* bad argument (maps to ValueError) */
    EPID_ERR_UNSUPPORTED = -4,    /* size / dtype outside what the kernels support */
    EPID_ERR_NOMEM = -5,
    EPID_ERR_NCCL = -6
};

/* element types of image batches (numpy dtypes the reference's operators preserve, core/array_utils.py) */
enum { EPID_U8 = 0, EPID_U16 = 1, EPID_I32 = 2, EPID_F32 = 3, EPID_F64 = 4, EPID_I16 = 5, EPID_I64 = 6 };

typedef struct epid_ctx epid_ctx;     /* one per device: stream(s), scratch, optional NCCL communicator */
typedef struct epid_batch epid_batch; /* n frames resident in HBM */

/* ----------------------------------------------------------------------------------------- context */
int32_t epid_device_count(int32_t* count);                    /* EPID_OK with *count == 0 if no GPU */
int32_t epid_ctx_create(int32_t device, epid_ctx** out);
int32_t epid_ctx_destroy(epid_ctx* ctx);
const char* epid_last_error(void);                             /* thread-local message of the last failure */
int32_t epid_sync(epid_ctx* ctx);
int32_t epid_device_info(epid_ctx* ctx, int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor, size_t* hbm_bytes);
/* PCI bus id ("0000:1b:00.0") of CUDA device `device`: lets a rank bind its host threads / pinned allocations to the GPU's NUMA node */
int32_t epid_device_pci_bus_id(int32_t device, char* out, int32_t cap);
int32_t epid_launch_count(epid_ctx* ctx, int64_t* launches);   /* kernels launched by this ctx so far */
int32_t epid_version(void);
/* options / diagnostic counters (no reference counterpart: the reference has a single CPU code path).
 * EPID_OPT_PF_EXACT_ONLY: 1 = always use the exact-histogram PicketFence pipeline (default 0: fused sample-guided front
 * kernel with automatic per-batch fallback to the exact pipeline).  EPID_CTR_PF_FALLBACKS: batches / chunks re-run exactly. */
enum { EPID_OPT_PF_EXACT_ONLY = 1,
       EPID_OPT_PF_WIN2 = 3 /* 1 (default) = two-kernel window path (medians + per-window analysis); 0 = single per-window kernel, kept as the
                               bit-exact reference for the two-kernel path */,
       EPID_OPT_STATS_EXACT = 7 /* 1: FieldAnalysis / Starshot compute check_inversion_by_histogram from the exact histogram for every frame
                                   (default 0: decision certified from exact counts at pilot thresholds, exact histogram only where that fails) */ };
enum { EPID_CTR_PF_FALLBACKS = 1, EPID_CTR_PF_REDONE_FRAMES = 2 /* frames re-run individually (fast re-run or exact pipeline) */,
       EPID_CTR_PF_EXACT_FRAMES = 3 /* of those: frames that went through the exact-histogram pipeline */,
       EPID_CTR_STATS_UNCERTIFIED = 4 /* FieldAnalysis / Starshot frames whose check_inversion_by_histogram decision needed exact percentiles */ };
int32_t epid_set_option(epid_ctx* ctx, int32_t key, int64_t value);
int32_t epid_get_counter(epid_ctx* ctx, int32_t key, int64_t* value);

/* pinned host memory (for the H2D legs of the batched entry points) */
int32_t epid_host_alloc(size_t bytes, void** out);
int32_t epid_host_free(void* p);

/* ----------------------------------------------------------------------------------------- batches */
/* replaces: ArrayImage(array) / DicomImage pixel_array  (core/image.py:1818-1848, 1431-1444) */
int32_t epid_batch_upload(epid_ctx* ctx, const void* host, int32_t dtype, int32_t n, int32_t h, int32_t w, epid_batch** out);
int32_t epid_batch_alloc(epid_ctx* ctx, int32_t dtype, int32_t n, int32_t h, int32_t w, epid_batch** out);
int32_t epid_batch_download(epid_batch* b, void* host);        /* whole batch, native dtype */
int32_t epid_batch_write(epid_batch* b, const void* host);     /* overwrite an existing batch from host memory (same shape / dtype) */
int32_t epid_batch_free(epid_batch* b);
int32_t epid_batch_shape(const epid_batch* b, int32_t* dtype, int32_t* n, int32_t* h, int32_t* w);
int32_t epid_batch_device_ptr(const epid_batch* b, void** dptr);

/* ----------------------------------------------------------------------------------------- frame statistics
 * One streaming read of every frame: min, max, sum, row sums, column sums, exact order statistics.
 * replaces: array.min()/max()/mean() (core/image.py:851,896; picketfence.py:231-232), np.percentile / np.median
 * of a full frame (picketfence.py:233,1510; core/image.py:918-920; winston_lutz.py:709,775; starshot.py:227,286),
 * np.sum/np.mean(image, axis) (picketfence.py:748-750,1513-1514; field_analysis.py:488-506).
 * The view [r0:r0+vh, c0:c0+vw] of each frame is analysed (crop is a view: core/image.py:714-745).
 * Integer dtypes U8/U16 only (exact integer histogram); q in percent, numpy 'linear' method.
 * Outputs (host, may be NULL): min,max: double[n]; sum: double[n] (exact integer sums < 2^53);
 * rowsum: double[n*vh] (sum over columns of each row); colsum: double[n*vw]; pct: double[n*nq]. */
int32_t epid_frame_stats(epid_ctx* ctx, const epid_batch* b, int32_t r0, int32_t c0, int32_t vh, int32_t vw,
                         const double* q_percent, int32_t nq,
                         double* mn, double* mx, double* sum, double* rowsum, double* colsum, double* pct);
/* full 65536-bin histogram of the view (uint32 counts [n][65536]); U8/U16 only */
int32_t epid_frame_histogram(epid_ctx* ctx, const epid_batch* b, int32_t r0, int32_t c0, int32_t vh, int32_t vw, uint32_t* hist);

/* ----------------------------------------------------------------------------------------- element-wise operators
 * All write a NEW batch (the reference rebinds self.array to a fresh ndarray, core/image.py:712,757,798,852,866). */
/* array_utils.invert  (core/array_utils.py:75-77): -a + max + min in the array's own dtype (modular for uints) */
int32_t epid_invert(epid_ctx* ctx, const epid_batch* in, epid_batch** out);
/* array_utils.bit_invert (core/array_utils.py:81-89): integer dtypes only, else EPID_ERR_INVALID */
int32_t epid_bit_invert(epid_ctx* ctx, const epid_batch* in, epid_batch** out);
/* array_utils.ground (core/array_utils.py:93-102): a - min + value, same dtype (value must be integral for integer
 * dtypes); mins (may be NULL): the n frame minima, in the batch's dtype */
int32_t epid_ground(epid_ctx* ctx, const epid_batch* in, double value, epid_batch** out, void* mins);
/* array_utils.normalize (core/array_utils.py:64-71): a / (value or max) -> F64; use_max != 0 ignores value */
int32_t epid_normalize(epid_ctx* ctx, const epid_batch* in, int32_t use_max, double value, epid_batch** out);
/* BaseImage.threshold (core/image.py:785-800): keep a >= t (kind 0, 'high') or a <= t (kind 1), else 0; same dtype */
int32_t epid_threshold(epid_ctx* ctx, const epid_batch* in, double t, int32_t kind, epid_batch** out);
/* BaseImage.as_binary (core/image.py:802-815): (a >= t) -> I64 0/1 */
int32_t epid_binarize(epid_ctx* ctx, const epid_batch* in, double t, epid_batch** out);

/* ----------------------------------------------------------------------------------------- stencils */
/* scipy.ndimage.median_filter(a, size=k) as called by array_utils.filter (core/array_utils.py:131):
 * full k x k footprint, mode='reflect', rank k*k/2, dtype preserved; frames of one row: the k-wide window at rank k/2.
 * EPID_ERR_UNSUPPORTED when the k-dependent tile exceeds the device's shared memory per block (DESIGN.md 4.7). */
int32_t epid_median_filter(epid_ctx* ctx, const epid_batch* in, int32_t size, epid_batch** out);
/* scipy.ndimage.gaussian_filter(a, sigma) as called by array_utils.filter (core/array_utils.py:133):
 * separable, axis 0 then axis 1, radius int(4*sigma+0.5), mode='reflect', float64 accumulate,
 * result of EACH pass cast to the input dtype (truncation for integers). */
int32_t epid_gaussian_filter(epid_ctx* ctx, const epid_batch* in, double sigma, epid_batch** out);
/* Same passes with caller-supplied correlate1d weights (2*radius+1 doubles).  The python binding passes the weights
 * scipy itself computes (scipy/ndimage/_filters.py:_gaussian_kernel1d) so integer results are bit-exact.
 * axes: 3 = axis 0 then axis 1 (2-D image), 1 = axis 0 only, 2 = axis 1 only (1-D profile stored as one row). */
int32_t epid_correlate1d_passes(epid_ctx* ctx, const epid_batch* in, const double* weights, int32_t radius, int32_t axes, epid_batch** out);
/* scipy.ndimage.sobel(a, axis) (core/image.py:1006-1007, BaseImage.gamma): reflect, same dtype semantics; out F32/F64 */
int32_t epid_sobel(epid_ctx* ctx, const epid_batch* in, int32_t axis, epid_batch** out);

/* ----------------------------------------------------------------------------------------- 1-D profiles
 * pylinac.core.profile.find_peaks (core/profile.py:2545-2649) == scipy.signal.find_peaks(height, distance,
 * prominence, width=min_width, rel_height = 1 - fwxm_height) + search-region trimming + top-max_number selection.
 * values: host double[n].  Arguments follow the reference's python signature after _parse_peak_args has NOT yet
 * been applied (threshold in [0,1] is a ratio of the range, separation in [0,1] a ratio of len, region <= 1 ratios).
 * peak_sort: 0 = 'prominences', 1 = 'peak_heights'.  required_prominence < 0: none.  max_number: EPID_PEAKS_ALL keeps every
 * peak (python None); any other value k keeps [:k] of the peaks in descending peak_sort order, as the reference slices: 0 keeps
 * none, -k all but the k smallest.  Equal keys rank the right-most peak first.  fwxm_height > 1 is EPID_ERR_INVALID (scipy's
 * negative rel_height).
 * Outputs (capacity cap each): idx int64; heights, prominences, left_bases(int64), right_bases(int64), widths,
 * width_heights, left_ips, right_ips double.  *count = number of peaks returned. */
#define EPID_PEAKS_ALL INT32_MIN
typedef struct {
    double threshold;           /* -inf allowed */
    double peak_separation;
    int32_t max_number;
    double fwxm_height;         /* 0..1 */
    double min_width;
    double search_lo, search_hi;
    int32_t peak_sort;
    double required_prominence; /* < 0: None */
} epid_peak_params;

int32_t epid_find_peaks(epid_ctx* ctx, const double* values, int32_t n, const epid_peak_params* p, int32_t cap,
                        int64_t* idx, double* heights, double* prominences, int64_t* left_bases, int64_t* right_bases,
                        double* widths, double* width_heights, double* left_ips, double* right_ips, int32_t* count);

/* ----------------------------------------------------------------------------------------- Picket Fence
 * PicketFence(image).analyze(**params) + the scalar set of results_data()  (picketfence.py:209-219, 280-329,
 * 636-912, 1313-1363, 1501-1743, 1857-1923) for a batch of frames, one result per frame. */
#define EPID_PF_MAX_PICKETS 32
#define EPID_PF_MAX_LEAVES 160

enum { /* per-frame status (maps to the reference's exceptions) */
    EPID_PF_OK = 0,
    EPID_PF_NO_PICKETS = 1,        /* ValueError "No pickets were found" (picketfence.py:760-764) */
    EPID_PF_NO_MEASUREMENTS = 2,   /* ValueError "No MLC measurements were found" (picketfence.py:804-807) */
    EPID_PF_TOO_MANY_PICKETS = 3,  /* more than EPID_PF_MAX_PICKETS peaks (unsupported) */
    EPID_PF_WINDOW_NO_PEAK = 4,    /* reference would raise IndexError inside FWXMProfile.field_edge_idx */
    EPID_PF_CAPACITY = 5,          /* measurement table capacity exceeded */
    EPID_PF_FLAT_IMAGE = 6,        /* max == min: the reference divides by zero */
    EPID_PF_EMPTY_FIT = 7,         /* a picket keeps no measurement, or a .5 median kiss count keeps no leaf row: the reference's
                                      np.polyfit of nothing raises TypeError (picketfence.py:810-828, 1881-1899) */
    EPID_PF_NAN_SPACING = 8        /* one picket and no picket_spacing: np.median(np.diff([i])) is nan and the reference raises
                                      ValueError "cannot convert float NaN to integer" in _get_mlc_window (picketfence.py:869-886) */
};

typedef struct {
    /* constructor (picketfence.py:280-329; PFDicomImage :209-219) */
    double dpmm;                 /* image.dpmm (core/image.py:1534-1547) */
    int32_t crop_px;             /* int(round(crop_mm * dpmm)) */
    int32_t filter_size;         /* median filter size, 0 = None */
    /* analyze() (picketfence.py:636-654) */
    double tolerance;
    double action_tolerance;     /* < 0: None */
    int32_t num_pickets;         /* 0: None */
    int32_t sag_px;              /* int(round(sag_adjustment * dpmm)) */
    int32_t orientation;         /* -1 auto, 0 Up-Down, 1 Left-Right */
    int32_t invert;
    double leaf_analysis_width_ratio;
    double picket_spacing;       /* < 0: None (auto) */
    double height_threshold;
    double edge_threshold;
    int32_t peak_sort;           /* 0 'prominences', 1 'peak_heights' */
    double required_prominence;
    int32_t separate_leaves;
    double nominal_gap_mm;
    int32_t has_cax_override;    /* PFDicomImage.center override (picketfence.py:246-260) */
    double cax_x_px, cax_y_px;   /* final centre in pixels when has_cax_override */
    /* MLC arrangement (picketfence.py:68-135): centres (mm), widths (mm), leaf numbers, in the reference's order */
    int32_t n_leaves;
    double leaf_center_mm[EPID_PF_MAX_LEAVES];
    double leaf_width_mm[EPID_PF_MAX_LEAVES];
    int32_t leaf_num[EPID_PF_MAX_LEAVES];
} epid_pf_params;

typedef struct { /* one per frame */
    int32_t status;
    int32_t orientation;                 /* 0 Up-Down, 1 Left-Right */
    int32_t noise_median_passes;         /* how often _check_for_noise filtered (picketfence.py:221-227) */
    int32_t corner_inverted;             /* check_inversion fired (core/image.py:868-897) */
    int32_t height, width;               /* analysed (cropped) shape */
    int32_t n_pickets;
    int32_t n_meas;                      /* rows of the measurement table that belong to this frame (after pruning) */
    int32_t n_leaves_removed;            /* leaf rows dropped by the median-count rule (picketfence.py:810-828) */
    int32_t passed;
    int32_t max_error_picket;
    int32_t max_error_leaf;              /* leaf number; for separate_leaves bank in max_error_bank (0 = A, 1 = B) */
    int32_t max_error_bank;
    int32_t n_failed;                    /* number of failing measurements (see table 'passed' flags) */
    double picket_spacing_px;
    double percent_passing;
    double max_error_mm;
    double abs_median_error_mm;
    double mean_picket_spacing_mm;
    double mlc_skew;
    double cax_px;                       /* image.center component along leaf travel */
    int32_t picket_idx[EPID_PF_MAX_PICKETS];      /* find_fwxm_peaks indices (bit-exact target) */
    double picket_val[EPID_PF_MAX_PICKETS];
    double fit_slope[EPID_PF_MAX_PICKETS];        /* np.polyfit(deg 1) of each picket */
    double fit_intercept[EPID_PF_MAX_PICKETS];
    double offsets_from_cax_mm[EPID_PF_MAX_PICKETS];
    double picket_width_max[EPID_PF_MAX_PICKETS]; /* picket_width_stat (picketfence.py:471-491) */
    double picket_width_mean[EPID_PF_MAX_PICKETS];
    double picket_width_median[EPID_PF_MAX_PICKETS];
    double picket_width_min[EPID_PF_MAX_PICKETS];
} epid_pf_summary;

typedef struct { /* one per kept MLCValue, leaf-major / picket-minor like PicketFence.mlc_meas */
    int32_t leaf_num;
    int32_t picket;
    int32_t passed[2];
    double position[2];      /* px along leaf travel; [1] only for separate_leaves */
    double error[2];         /* mm */
    double width_mm;         /* profile.field_width_mm */
} epid_pf_meas;

/* device-resident batch (uint16): results to host.  meas: [n][meas_cap].  Synchronous. */
int32_t epid_pf_analyze(epid_ctx* ctx, const epid_batch* frames, const epid_pf_params* p,
                        epid_pf_summary* summary, epid_pf_meas* meas, int32_t meas_cap);
/* end-to-end: host frames [n][h][w] uint16 (pinned or pageable) -> chunked H2D overlapped with compute -> results. */
int32_t epid_pf_analyze_host(epid_ctx* ctx, const uint16_t* frames, int32_t n, int32_t h, int32_t w,
                             const epid_pf_params* p, epid_pf_summary* summary, epid_pf_meas* meas, int32_t meas_cap);
/* timing hooks for bench.py: run the device-resident pipeline `iters` times back to back (results stay on the
 * device except the last), return the CUDA-event time of the whole region and of the frame-statistics kernel. */
int32_t epid_pf_bench(epid_ctx* ctx, const epid_batch* frames, const epid_pf_params* p, int32_t iters,
                      float* total_ms, float* stats_kernel_ms, int64_t* launches);
/* the same timed region with CUDA-event marks between the kernels: total_ms of `iters` back-to-back passes, stage_ms[k] summed over
 * the passes (stage ids as for epid_pf_bench_stages), kernel launches and the number of frames the per-frame exact fallback re-ran
 * (when the batch contains deferred frames the passes are timed with the host round trip of the fallback included) */
int32_t epid_pf_bench_timed(epid_ctx* ctx, const epid_batch* frames, const epid_pf_params* p, int32_t iters, float* total_ms,
                            float* stage_ms, int32_t nstages, int64_t* launches, int64_t* redone_frames);
/* per-stage device times of `iters` passes (CUDA events between the kernels; bench.py's per-kernel roofline table):
 * stage_ms[0..8] = init + pilot, stream, tail, windows (per-window kernel), windows (generic), finalize, exact front end (fallback
 * only), windows (two-kernel path: medians), windows (two-kernel path: per-window analysis) */
int32_t epid_pf_bench_stages(epid_ctx* ctx, const epid_batch* frames, const epid_pf_params* p, int32_t iters, float* stage_ms,
                             int32_t nstages);


/* ----------------------------------------------------------------------------------------- Starshot
 * Starshot(image).analyze(**params)  (starshot.py:105-125, 197-401, 701-834; CollapsedCircleProfile core/profile.py:
 * 2244-2283, 2405-2483) for a batch of uint16 frames, one result per frame. */
#define EPID_STAR_MAX_PEAKS 64

enum { /* per-frame status (maps to the reference's exceptions) */
    EPID_STAR_OK = 0,
    EPID_STAR_NO_WOBBLE = 1,       /* RuntimeError "unable to determine a reasonable wobble" (starshot.py:372-376) */
    EPID_STAR_NO_LINES = 2,        /* RuntimeError "unable to properly detect the radiation lines" (starshot.py:339-342) */
    EPID_STAR_NO_START_POINT = 3,  /* no FW80M peak in the central third (reference: IndexError) */
    EPID_STAR_CAPACITY = 4,        /* profile / peak capacity exceeded */
    EPID_STAR_FLAT_IMAGE = 5
};

typedef struct {
    double dpmm;                  /* image.dpmm */
    double radius;                /* analyze() arguments (starshot.py:230-240) */
    double min_peak_height;
    double max_wobble_diameter;
    double tolerance;
    int32_t has_start_point;
    double start_x, start_y;
    int32_t fwhm;
    int32_t recursive;
    int32_t invert;
} epid_star_params;

typedef struct { /* one per frame */
    int32_t status;
    int32_t hist_inverted;        /* check_inversion_by_histogram([4, 50, 96]) fired */
    int32_t start_x, start_y;     /* _get_reasonable_start_point (bit-exact target) */
    double local_max;             /* np.percentile(central third, 90) */
    int32_t iterations;           /* StarProfile constructions of _get_reasonable_wobble */
    int32_t profile_len;
    double radius_px;             /* circle_profile.radius */
    int32_t n_peaks, n_lines;
    int32_t peak_idx[EPID_STAR_MAX_PEAKS];   /* find_fwxm_peaks indices on the rolled profile (bit-exact target) */
    double peak_x[EPID_STAR_MAX_PEAKS], peak_y[EPID_STAR_MAX_PEAKS];
    double wobble_x, wobble_y;    /* wobble.center (px) */
    double wobble_radius_px, wobble_radius_mm;
    double angles[EPID_STAR_MAX_PEAKS / 2];
    int32_t passed;
    int32_t pad;
} epid_star_result;

/* gauss_weights / gauss_offsets: scipy _gaussian_kernel1d tables for sigma = 1 .. max_sigma (host; weights of sigma s start at
 * gauss_offsets[s], 2 * int(4 s + 0.5) + 1 doubles each), computed by the binding exactly like scipy does. */
int32_t epid_starshot_analyze(epid_ctx* ctx, const epid_batch* frames, const epid_star_params* p, const double* gauss_weights,
                              const int32_t* gauss_offsets, int32_t max_sigma, epid_star_result* results);


/* CircleProfile / CollapsedCircleProfile._profile + x / y locations (core/profile.py:2179-2283, 2405-2483) of ONE image
 * (batch of 1; U8 / U16 / F32 / F64): nearest-neighbour samples (scipy.ndimage.map_coordinates order=0, 0 outside) on
 * radians = arange(start_angle, 2 pi + start_angle - interval, interval)[::-1 if ccw], interval = 2 pi / (pi * r_max * 2 *
 * sampling_ratio); collapsed != 0: mean over num_profiles radii linspace(r (1 - width_ratio), r (1 + width_ratio)).
 * cap: capacity of the three output arrays; *count = number of samples. */
int32_t epid_circle_profile(epid_ctx* ctx, const epid_batch* image, double cx, double cy, double radius, double start_angle,
                            int32_t ccw, double sampling_ratio, int32_t collapsed, double width_ratio, int32_t num_profiles,
                            int32_t cap, double* profile, double* x_locations, double* y_locations, int32_t* count);

/* ----------------------------------------------------------------------------------------- Field analysis
 * FieldAnalysis(image).analyze(**params)  (field_analysis.py:445-864, 1069-1117; protocol functions :37-231; SingleProfile
 * core/profile.py:1125-1937) for a batch of uint16 frames, one result per frame.  Interpolation NONE / LINEAR, edge
 * detection FWHM / INFLECTION_DERIVATIVE, every normalisation, protocols NONE / VARIAN / SIEMENS / ELEKTA. */
enum { /* per-frame status */
    EPID_FIELD_OK = 0,
    EPID_FIELD_NO_EDGES = 1,     /* a profile without a usable peak / inflection (reference: IndexError in find_peaks output) */
    EPID_FIELD_FLAT_IMAGE = 2
};

typedef struct {
    double dpmm;                       /* image.dpmm */
    int32_t protocol;                  /* 0 NONE, 1 VARIAN, 2 SIEMENS, 3 ELEKTA (field_analysis.py:233-289) */
    int32_t centering;                 /* 0 MANUAL, 1 BEAM_CENTER, 2 GEOMETRIC_CENTER (core/profile.py:187-192) */
    double vert_position, horiz_position, vert_width, horiz_width;
    double in_field_ratio, slope_exclusion_ratio;
    int32_t invert;
    double penumbra_lower, penumbra_upper;
    int32_t interpolation;             /* 0 NONE, 1 LINEAR */
    double interpolation_resolution_mm;
    int32_t ground;
    int32_t normalization;             /* 0 NONE, 1 GEOMETRIC_CENTER, 2 BEAM_CENTER, 3 MAX */
    int32_t edge;                      /* 0 FWHM, 1 INFLECTION_DERIVATIVE */
    double edge_smoothing_ratio;
} epid_field_params;

typedef struct { /* one per frame: FieldAnalysis._results + protocol results (field_analysis.py:755-863) */
    int32_t status;
    int32_t hist_inverted;             /* check_inversion_by_histogram() fired (field_analysis.py:472) */
    int32_t strip_rows[2];             /* rows [bottom, top) averaged into the horizontal profile */
    int32_t strip_cols[2];             /* columns [left, right) averaged into the vertical profile */
    int32_t profile_len[2];            /* samples of the horizontal / vertical SingleProfile */
    double top_penumbra_mm, bottom_penumbra_mm, left_penumbra_mm, right_penumbra_mm;
    double geometric_center_index_x_y[2], beam_center_index_x_y[2];
    double field_size_vertical_mm, field_size_horizontal_mm;
    double beam_center_to_top_mm, beam_center_to_bottom_mm, beam_center_to_left_mm, beam_center_to_right_mm;
    double cax_to_top_mm, cax_to_bottom_mm, cax_to_left_mm, cax_to_right_mm;
    double top_position_index_x_y[2];
    double top_horizontal_distance_from_cax_mm, top_vertical_distance_from_cax_mm;
    double top_horizontal_distance_from_beam_center_mm, top_vertical_distance_from_beam_center_mm;
    double left_slope_percent_mm, right_slope_percent_mm, top_slope_percent_mm, bottom_slope_percent_mm;
    double symmetry_horizontal, symmetry_vertical, flatness_horizontal, flatness_vertical;
} epid_field_result;

/* samples of SingleProfile(values of length n0, dpmm, interpolation, resolution) (core/profile.py:1306-1322) */
int32_t epid_field_profile_len(int32_t n0, double dpmm, int32_t interpolation, double resolution_mm);
/* gauss_h / gauss_v: scipy gaussian_filter1d weights (2 * lw + 1 doubles, already reversed for correlate1d) for
 * sigma = edge_smoothing_ratio * profile length of the horizontal / vertical profile; may be NULL when edge == 0. */
int32_t epid_field_analyze(epid_ctx* ctx, const epid_batch* frames, const epid_field_params* p, const double* gauss_h, int32_t lw_h,
                           const double* gauss_v, int32_t lw_v, epid_field_result* results);

/* SingleProfile(values, dpmm, interpolation, ground, ..., edge_detection_method, ...) and its query methods for ONE host
 * profile (core/profile.py:1125-1937): fwxm_data(x), beam_center(), geometric_center(), inflection_data(), penumbra(lower,
 * upper), field_data(in_field_ratio, slope_exclusion_ratio), all evaluated in one launch.  Indices are in the units of the
 * original samples (x_values = range(len(values))); the interpolated abscissae are linspace(x_start, x_stop, n). */
typedef struct {
    double dpmm;                       /* <= 0: None (interpolation_factor is used) */
    int32_t interpolation;             /* 0 NONE, 1 LINEAR, 2 = values are already sampled on linspace(x_start, x_stop, n0): cubic
                                          (Interpolation.SPLINE) interpolation or custom uniform x_values, prepared by the caller */
    double interpolation_resolution_mm, interpolation_factor;
    int32_t ground, normalization, edge, centering;   /* codes as in epid_field_params; centering 2 = GEOMETRIC_CENTER; edge 2 = the
                                          field edges are supplied (edge_left / edge_right: Hill-function inflection points) */
    double edge_smoothing_ratio;
    double x_start, x_stop;            /* interpolation == 2 */
    double edge_left, edge_right;      /* edge == 2 */
} epid_sp_params;

typedef struct {
    int32_t status;                    /* 0 ok, 1: no usable peak while normalising */
    int32_t n;                         /* samples after interpolation */
    double x_start, x_stop;
    double values_max;
    double geometric_center_index, geometric_center_value;
    int32_t beam_ok, fwxm_ok, infl_ok, pen_ok, fd_ok, fd_field_values_n;
    double beam_center_index, beam_center_value_at_rounded;
    double fwxm_left, fwxm_right, fwxm_center_value_at_rounded, fwxm_left_value_at_rounded, fwxm_right_value_at_rounded;
    double infl_left, infl_right, infl_left_value_exact, infl_right_value_exact, infl_left_value_rounded, infl_right_value_rounded;
    double pen_left_lower, pen_left_upper, pen_right_lower, pen_right_upper;
    double fd_width, fd_beam_center, fd_cax, fd_left, fd_right, fd_inner_left, fd_inner_right;
    double fd_left_slope, fd_left_intercept, fd_right_slope, fd_right_intercept;
    double fd_top_index, fd_top_value, fd_top_params[3];
    double fd_beam_center_value, fd_cax_value, fd_left_value, fd_right_value;
} epid_sp_result;

/* x_values: NULL, or with interpolation == 2 the n0 increasing (possibly unevenly spaced) abscissae of `values` (x_start / x_stop are
 * then x_values[0] / x_values[n0 - 1]).  gauss: gaussian_filter1d weights for sigma = edge_smoothing_ratio * n_expect (NULL when edge == 0).  values_out (cap):
 * the interpolated / grounded / normalised values; field_values_out (cap): field_data()["field values"]. */
int32_t epid_single_profile(epid_ctx* ctx, const double* values, const double* x_values, int32_t n0, const epid_sp_params* p, const double* gauss, int32_t lw,
                            int32_t n_expect, double fwxm_x, double pen_lower, double pen_upper, double in_field_ratio,
                            double slope_exclusion_ratio, epid_sp_result* result, double* values_out, double* field_values_out,
                            int32_t cap);

/* ----------------------------------------------------------------------------------------- Winston-Lutz (per image)
 * WinstonLutz2D(image).analyze(bb_size_mm, low_density_bb, open_field, bb_proximity_mm) (winston_lutz.py:668-829, 1109-1231;
 * SizedDiskLocator / find_features metrics/image.py:564-612, metrics/utils.py:66-190; predicates metrics/features.py:7-68) for a
 * batch of uint16 frames, one result per frame.  BB arrangement ISO (nominal BB position = EPID centre), no shift vector. */
enum { /* per-frame status (maps to the reference's exceptions) */
    EPID_WL_OK = 0,
    EPID_WL_NO_BB = 1,        /* ValueError "Couldn't find the minimum number of disks" / BB_ERROR_MESSAGE */
    EPID_WL_MISMATCH = 2,     /* ValueError "The number of detected fields and BBs do not match" */
    EPID_WL_NO_FIELD = 3,     /* ValueError "No fields were detected" */
    EPID_WL_CAPACITY = 4,     /* search window / field / region larger than the kernels' shared-memory tiles */
    EPID_WL_FLAT_IMAGE = 5
};

typedef struct {
    double dpmm;
    double bb_size_mm;
    int32_t low_density_bb;
    int32_t open_field;
    double bb_proximity_mm;
} epid_wl_params;

typedef struct { /* one per frame */
    int32_t status;
    int32_t inverted;             /* check_inversion_by_histogram((0.01, 50, 99.99)) fired */
    int32_t crop_px;              /* pixels _clean_edges removed from every edge */
    int32_t height, width;        /* analysed (cropped) shape */
    int32_t n_bbs;                /* BB candidates accepted at the first successful threshold */
    int32_t threshold_passes;     /* thresholds visited by find_features */
    int32_t pad;
    double bb_x, bb_y;            /* matched BB (weighted centroid), pixels of the cropped image */
    double field_x, field_y;      /* field CAX (centre of mass of the filled field mask) */
    double epid_x, epid_y;        /* image centre */
    double cax2bb_x, cax2bb_y, cax2bb_distance;         /* mm */
    double cax2epid_x, cax2epid_y, cax2epid_distance;   /* mm */
} epid_wl_result;

int32_t epid_wl2d_analyze(epid_ctx* ctx, const epid_batch* frames, const epid_wl_params* p, epid_wl_result* results);

/* ----------------------------------------------------------------------------------------- SizedDiskRegion / SizedDiskLocator
 * img.compute(SizedDiskLocator(...)) (metrics/image.py:402-667): sample = image[window] around the expected position, inverted,
 * stretched to [0, 1]; find_features (metrics/utils.py:66-190): <= 50 thresholds { label (4-connectivity), clear_border, regionprops,
 * is_right_size_bb / is_round / is_right_circumference / is_symmetric / is_solid } -> weighted centroids, de-duplicated by the
 * minimum separation, until max_number points are found.  One result per uint16 frame; status values are EPID_WL_*. */
#define EPID_DISK_MAX 8
typedef struct {
    double dpmm;
    double expected_x, expected_y;     /* pixels, image coordinates (the caller has applied from_center / the physical-units quirks) */
    double window_w, window_h;         /* search window, pixels */
    double radius_mm, tolerance_mm;
    double min_separation_px;
    int32_t invert;
    int32_t max_number;
    int32_t conditions;                /* bit mask of the detection conditions: 1 is_right_size_bb, 2 is_round, 4 is_right_circumference,
                                          8 is_symmetric, 16 is_solid (metrics/features.py:7-68), 32 is_modest_size (winston_lutz.py:598-606) */
    int32_t pad;
} epid_disk_params;

typedef struct {
    int32_t status;
    int32_t n_points;                  /* detected disks (image coordinates x[], y[]) */
    int32_t n_regions;                 /* regions that passed every condition at the LAST threshold visited (what find_features returns) */
    int32_t passes;
    int32_t left, top;                 /* offsets of the sample window */
    double x[EPID_DISK_MAX], y[EPID_DISK_MAX];
    /* regionprops of those regions, sample (window) coordinates */
    double r_area[EPID_DISK_MAX], r_filled_area[EPID_DISK_MAX], r_perimeter[EPID_DISK_MAX], r_convex_area[EPID_DISK_MAX];
    double r_centroid_y[EPID_DISK_MAX], r_centroid_x[EPID_DISK_MAX], r_wcentroid_y[EPID_DISK_MAX], r_wcentroid_x[EPID_DISK_MAX];
    int32_t r_bbox[EPID_DISK_MAX][4];  /* min_row, min_col, max_row, max_col (half-open) */
} epid_disk_result;

int32_t epid_disk_locate(epid_ctx* ctx, const epid_batch* frames, const epid_disk_params* p, epid_disk_result* results);

/* ----------------------------------------------------------------------------------------- spline zoom
 * scipy.ndimage.zoom(a, zoom, order, mode) for 2-D frames (both axes) or 1-D profiles (h == 1: the sample axis) ->
 * float64 batch of shape round(shape * zoom).  order 1 or 3; mode 0 = 'constant' (equate_images, core/image.py:217), 1 = 'nearest'
 * (ProfileBase.as_resampled, core/profile.py:384-390), 3 = 'nearest' with grid_mode=True (PhysicalProfileMixin.as_resampled,
 * core/profile.py:951-1013). */
int32_t epid_zoom(epid_ctx* ctx, const epid_batch* in, double zoom, int32_t order, int32_t mode, epid_batch** out);

/* BaseImage.rotate(angle, mode) (core/image.py:780-783): skimage.transform.rotate(order 1) semantics -- img_as_float conversion
 * (uint8 / 255, uint16 / 65535), counter-clockwise rotation by angle_deg about (cols / 2 - 0.5, rows / 2 - 0.5), bilinear sampling;
 * mode 0 = 'constant' (0 outside), 1 = 'edge'.  float64 output of the input shape. */
int32_t epid_rotate(epid_ctx* ctx, const epid_batch* in, double angle_deg, int32_t mode, epid_batch** out);

/* ----------------------------------------------------------------------------------------- gamma map
 * BaseImage.gamma (core/image.py:928-1017), Bakai eq. 6: ref / comp are the float64 images AFTER the reference's inversion check,
 * ground() and normalize(); threshold_abs = threshold * max(ref); dose_frac = doseTA / 100; dist_px = distTA * dpmm.  The Sobel
 * gradient (scipy.ndimage.sobel on the float32 reference with nan below the threshold, mode reflect), hypot and the division are
 * one fused kernel; out: a new float64 batch (nan where the reference is below the threshold). */
int32_t epid_gamma(epid_ctx* ctx, const epid_batch* ref, const epid_batch* comp, double threshold_abs, double dose_frac, double dist_px,
                   epid_batch** out);
/* pylinac.core.gamma.gamma_2d (core/gamma.py:229-330), Low et al. 2004 Table I, for n (reference, evaluation) pairs: dose_frac =
 * dose_to_agreement / 100 times reference.max() (global_dose != 0, taken on the device per pair; a nan makes it nan) or times the
 * reference elementwise; threshold = dose_threshold / 100, compared with the normalised reference; pixels at or above it take the
 * minimum over the disk of dist2[k] + (eval_n - ref_n)^2 with the evaluation clamped to its own shape (np.pad mode 'edge'), capped
 * at cap (cap2 = cap**2 as the caller computes it); others take fill_value.  offsets: [n_off][2] (row, col) of skimage.draw.disk((0,
 * 0), dta + 1) and dist2 their (r / dta)**2 + (c / dta)**2, sorted by dist2, raster order breaking ties.  Any dtype; numpy 2
 * promotion (a float32 reference normalises in float32).  Global mode needs an evaluation at least the reference's shape, local mode
 * equal shapes.  full_search != 0 disables the exact early exit.  out: a new float64 batch of the reference's shape, bit-identical to
 * the reference. */
int32_t epid_gamma2d(epid_ctx* ctx, const epid_batch* ref, const epid_batch* eval, double dose_frac, double threshold, double cap,
                     double cap2, double fill_value, int32_t global_dose, const int32_t* offsets, const double* dist2, int32_t n_off,
                     int32_t full_search, epid_batch** out);
/* pylinac.core.gamma.gamma_geometric (core/gamma.py:105-226, Ju et al. 2008) for n profile pairs, all arrays in host memory.  Pair i
 * has the normalised evaluation samples eval_x / eval_y[eval_off[i] .. eval_off[i + 1]] (strictly monotonic x, decreasing[i] != 0 when
 * decreasing, at least 2 samples when the pair has points) and the normalised evaluated reference points ref_x / ref_y[pt_off[i] ..
 * pt_off[i + 1]].  dta is the distance to agreement the reference subtracts from the normalised x, cap the gamma cap.  gamma[k]: the
 * capped minimum segment distance of point k, bit-identical to the reference; svd_fail[i] != 0 where a segment of pair i has a nan
 * V^T V (the reference's pinv raises LinAlgError).  One upload, one kernel, one download. */
int32_t epid_gamma_geometric(epid_ctx* ctx, int32_t n, const int64_t* eval_off, const int64_t* pt_off, const int32_t* decreasing,
                             const double* eval_x, const double* eval_y, const double* ref_x, const double* ref_y, double dta, double cap,
                             double* gamma, int32_t* svd_fail);
/* pylinac.core.gamma.gamma_1d (core/gamma.py:333-460, Low et al. 2004) for n profile pairs, all arrays in host memory: eval_x / eval_y
 * are each pair's evaluation coordinates and values sorted by x (interp1d's stable sort; at least 2 when the pair has points), ref_x /
 * ref_y the evaluated reference points, dose_ta2[k] the dose criterion squared of point k (float32 values where dose_f32[i] != 0: the
 * dose term then divides in float32).  Each point samples np.linspace(ref_x - dta, ref_x + dta, num), interpolates the evaluation
 * there (interp1d linear, extrapolating) and takes min sqrt(dist**2 / dta2 + dose**2 / dose_ta2), capped at cap.  Outputs gamma[k],
 * samples[k * num + j] and sample_x[k * num + j].  One upload, one kernel, one download. */
int32_t epid_gamma1d(epid_ctx* ctx, int32_t n, const int64_t* eval_off, const int64_t* pt_off, const int32_t* dose_f32, const double* eval_x,
                     const double* eval_y, const double* ref_x, const double* ref_y, const double* dose_ta2, double dta, double dta2,
                     int32_t num, double cap, double* gamma, double* samples, double* sample_x);

/* ----------------------------------------------------------------------------------------- ROI statistics / weighted centroid
 * RectangleROI.mean / std / min / max (core/roi.py:533-706): pixels of a rectangle given by its corners verts_xy[nroi][4][(x, y)]
 * (any rotation), selected like skimage.draw.polygon (pixel centres inside or on the boundary, clipped to the image).  Every ROI is
 * evaluated on every frame of the batch: outputs [n][nroi] (may be NULL).  std is the population standard deviation (np.std). */
int32_t epid_roi_stats(epid_ctx* ctx, const epid_batch* b, int32_t nroi, const double* verts_xy, double* count, double* mean,
                       double* std, double* mn, double* mx);
/* WeightedCentroid.calculate (metrics/image.py:959-983): cx = sum(x * a) / sum(a), cy likewise; total = sum(a) (may be NULL). */
int32_t epid_weighted_centroid(epid_ctx* ctx, const epid_batch* b, double* cx, double* cy, double* total);
/* DiskROI / HighContrastDiskROI statistics (core/roi.py:39-190, 411-478): for disk i, disks[i] = (frame index, centre row, centre
 * column, radius), the pixels arr[skimage.draw.disk((cy, cx), r)] of that frame of the batch (raster order; negative indices wrap as
 * numpy's fancy indexing does) -> count / mean / std / min / max / median [ndisk] (any may be NULL), each equal bit for bit to
 * np.mean / np.std / np.min / np.max / np.median of those pixels.  Any dtype.  An empty disk has count 0 and NaN elsewhere; a NaN pixel
 * makes min, max and median NaN.  A member pixel at or beyond the frame's size (numpy's IndexError) returns EPID_ERR_INVALID; a bounding
 * box of more than 16384 rows or columns EPID_ERR_UNSUPPORTED. */
int32_t epid_disk_stats(epid_ctx* ctx, const epid_batch* b, int32_t ndisk, const double* disks, double* count, double* mean,
                        double* std, double* mn, double* mx, double* median);
/* LowContrastDiskROI.percentile (core/roi.py:406-408): out[i * nq + k] = np.percentile(arr[skimage.draw.disk((cy, cx), r)], q_percent[k])
 * (method "linear") of disk i, disks as for epid_disk_stats, equal bit for bit to numpy's for q_percent[k] passed as a Python number:
 * the value of a float32 batch is numpy's float32 result, widened.  1 <= nq <= 16.  A disk with a NaN pixel, or an empty disk, gives
 * NaN (numpy raises IndexError for an empty one).  A q_percent outside [0, 100] (checked as numpy does, in float32 for a float32 batch)
 * returns EPID_ERR_INVALID with numpy's message; a member pixel beyond the frame returns EPID_ERR_INVALID. */
int32_t epid_disk_percentiles(epid_ctx* ctx, const epid_batch* b, int32_t ndisk, const double* disks, int32_t nq, const double* q_percent,
                              double* out);

/* ----------------------------------------------------------------------------------------- VMAT (DRGS / DRMLC) and DLG
 * VMATBase.__init__ / analyze, VMATLinearBase._identify_images / _roi_profiles / _calculate_segments, Segment.r_corr / stdev,
 * _update_r_corrs (vmat.py:249-275, 309-346, 408-436, 739-841): n independent (image 1, image 2) pairs, img1->n == img2->n, uint16.
 * Per pair on the device: ground() + check_inversion() of both images (folded into an affine map of the raw pixels, nothing is
 * rewritten), column-mean FWXM profiles (ground, beam-centre normalisation, stretch, 90th-percentile normalisation, in-field
 * length / std) -> which image is the open field, field centre (image centre + warning flag when it lies outside the central
 * third), then per segment the mean / std of DMLC / open over the pixels of the segment rectangle (never materialising the ratio
 * image) -> R_corr, R_dev, pass / fail and the aggregates. */
#define EPID_VMAT_MAX_SEG 16
typedef struct {
    int32_t ground;              /* VMATBase(ground=True) */
    int32_t check_inversion;     /* VMATBase(check_inversion=True) */
    int32_t invert_image_order;  /* analyze(invert_image_order=False) */
    int32_t nseg;                /* len(roi_config) <= EPID_VMAT_MAX_SEG */
    double dpmm;
    double tolerance_percent;    /* analyze(tolerance=1.5) */
    double seg_w_mm, seg_h_mm;   /* segment_size_mm: (5, 100) */
    double offset_mm[EPID_VMAT_MAX_SEG];
} epid_vmat_params;

typedef struct {
    int32_t status;              /* 0 ok; 2: a column-mean profile has no peak (the reference raises IndexError) */
    int32_t open_is_first;       /* 1: image 1 is the open field (after invert_image_order) */
    int32_t inverted[2];         /* check_inversion() flipped image 1 / 2 */
    int32_t center_warning;      /* field centre outside the central third: image centre used (the reference warns) */
    int32_t passed;
    int32_t nseg;
    int32_t pad_;
    double x_field_center;
    double profile_center_idx[2];                 /* FWXM centre of the column-mean profile of image 1 / 2 */
    double field_len[2], field_std[2];            /* len / np.std of field_values() of image 1 / 2 */
    double r_corr[EPID_VMAT_MAX_SEG], r_dev[EPID_VMAT_MAX_SEG], stdev[EPID_VMAT_MAX_SEG];
    double center_x[EPID_VMAT_MAX_SEG], center_y[EPID_VMAT_MAX_SEG], npix[EPID_VMAT_MAX_SEG];
    int32_t seg_passed[EPID_VMAT_MAX_SEG];
    double max_r_deviation, avg_abs_r_deviation, avg_r_deviation;
} epid_vmat_row;
int32_t epid_vmat_analyze(epid_ctx* ctx, const epid_batch* img1, const epid_batch* img2, const epid_vmat_params* p,
                          epid_vmat_row* rows /* [n] host */);

/* element-wise true division num / den -> a new float64 batch (`dmlc_image.array / open_image.array`, vmat.py:339; x / 0 = inf,
 * 0 / 0 = nan like numpy); both uint16 or both float64, same shape.  Each frame is first mapped by v -> sign * v + offset
 * (sign_off[2 * (2 * i + which)] = sign, [.. + 1] = offset, which = 0 num / 1 den; NULL = identity): the ground() / invert() the
 * reference applied to the images before dividing. */
int32_t epid_divide(epid_ctx* ctx, const epid_batch* num, const epid_batch* den, const double* sign_off, epid_batch** out);

/* DLG.analyze (dlg.py:32-86, 112-127): per frame and per leaf window [bottom[l]:top[l], c0:c1] the column-mean profile, the
 * inversion rule of _determine_measured_gap and the prominence of its largest peak (signed) -> measured[n][nleaf]; then
 * scipy.stats.linregress(planned, measured) per frame -> slope, intercept, dlg = intercept / slope.  uint16 frames. */
int32_t epid_dlg_analyze(epid_ctx* ctx, const epid_batch* b, int32_t nleaf, const int32_t* bottom, const int32_t* top, int32_t c0,
                         int32_t c1, const double* planned, double* measured, double* slope, double* intercept, double* dlg);

/* ----------------------------------------------------------------------------------------- whole-frame feature finders
 * GlobalSizedDiskLocator.calculate (metrics/image.py:329-354 -> find_features, metrics/utils.py:66-190) and GlobalSizedFieldLocator /
 * GlobalFieldLocator.calculate (metrics/image.py:817-897): the whole frame is binarised at the reference's rising thresholds,
 * labelled (4-connectivity for disks, 8 for fields), cleared at the border and every region is put through the detection conditions.
 * The device returns every region that passed, for every threshold, ordered like the reference visits them (threshold, then label);
 * the reference's point de-duplication / stop rule (which depends on what was found so far) is scalar work on these records in the
 * binding.  uint16 frames. */
typedef struct {
    int32_t mode;            /* 0: find_features (stretch(invert?(array)), cutoffs imin + k * step, k = 1..), 1: field locator (array as is,
                                cutoffs imin + (5 + k) * step) */
    int32_t invert;          /* mode 0: GlobalSizedDiskLocator(invert=True) */
    int32_t sample_kind;     /* 0: image.array is the integer frame; 1: image.array is the ground()-ed + normalize()-d float image of the
                                frame (Winston-Lutz images after analyze()) */
    int32_t conditions;      /* bit mask: 1 is_right_size_bb, 2 is_round, 4 is_right_circumference, 8 is_symmetric, 32 is_modest_size,
                                64 is_square, 128 is_right_square_size, 256 is_right_square_perimeter, 512 is_right_area_square
                                (metrics/features.py, winston_lutz.py:598-621) */
    double dpmm;
    double radius_mm, tolerance_mm;                              /* bb_size / tolerance of the disk conditions */
    double field_width_mm, field_height_mm, field_tolerance_mm;  /* field conditions */
    double bb_size_mm, rad_size_mm;                              /* is_modest_size / is_right_square_size */
} epid_locate_params;

typedef struct {
    int32_t threshold_index;     /* 0-based position of the threshold in the reference's sweep */
    int32_t label_root;          /* raster index of the region's first pixel (= order of skimage's labels) */
    int32_t bbox[4];             /* min_row, min_col, max_row, max_col (half-open) */
    double area, area_filled, perimeter, equivalent_diameter;
    double centroid_y, centroid_x, wcentroid_y, wcentroid_x;
} epid_region;

/* regions: [n][region_cap]; counts[n]: accepted regions per frame; flags[n]: 1 = more candidates than the device list holds at some
 * threshold, 2 = more accepted regions than region_cap */
int32_t epid_global_locate(epid_ctx* ctx, const epid_batch* frames, const epid_locate_params* p, epid_region* regions, int32_t region_cap,
                           int32_t* counts, int32_t* flags);

/* ----------------------------------------------------------------------------------------- Canny / Hough (JawOrthogonality)
 * contrib/orthogonality.py:29-50: skimage.feature.canny(stretch(image)) -> skimage.transform.hough_line -> hough_line_peaks.
 * scikit-image is absent from the build container: restated from the published algorithms, parity unpinned (oracle/edges_oracle.py).
 * epid_canny: float64 frames; weights = scipy's gaussian kernel (2 * radius + 1 doubles) for the smoothing sigma; thresholds are
 * absolute (skimage defaults for float images: 0.1 / 0.2) -> uint8 edge maps (a new batch).
 * epid_hough_line: one uint8 edge map, ntheta angles (radians) -> int32 accumulator batch [1][2 * offset + 1][ntheta], offset =
 * ceil(hypot(rows, cols)); the distance bins are linspace(-offset, offset, 2 * offset + 1).
 * epid_hough_candidates: the device half of hough_line_peaks / _prominent_peaks: maximum filter (2 d + 1 per axis, mode 'constant'),
 * pixels equal to their local maximum and > threshold (threshold < 0: 0.5 * max) as (row, col, value) triples; `filtered` keeps the
 * max-filtered accumulator on the device for epid_gather_i32 (values at arbitrary (row, col) pairs). */
int32_t epid_canny(epid_ctx* ctx, const epid_batch* in, const double* weights, int32_t radius, double low_threshold, double high_threshold,
                   epid_batch** out);
int32_t epid_hough_line(epid_ctx* ctx, const epid_batch* edges, int32_t ntheta, const double* theta, epid_batch** accum, int32_t* offset_out);
int32_t epid_hough_candidates(epid_ctx* ctx, const epid_batch* accum, int32_t min_xdistance, int32_t min_ydistance, double threshold,
                              int32_t cap, int32_t* cand_yxv, int32_t* count, int32_t* global_max, epid_batch** filtered);
int32_t epid_gather_i32(epid_ctx* ctx, const epid_batch* img, int32_t npts, const int32_t* yx, int32_t* values);

/* ----------------------------------------------------------------------------------------- Varian XIM pixel decode
 * XIM._parse_lookup_table / _parse_compressed_bytes / _get_diffs (core/image.py:1186-1309) for a batch of n files that share
 * h x w and bytes_per_pixel.  arena: host memory (page-locked for a DMA copy; 16-byte aligned) holding every file's lookup table
 * and compressed pixel buffer; desc[f] = {lookup offset, lookup bytes, pixel offset, pixel bytes} (int64 [n][4], offsets 16-byte
 * aligned, inside the arena).  One H2D copy of the arena and one launch sequence for the whole batch.
 * dtype: the reference's dtype (EPID_I16 for bpp 1 and 2 -- bpp 1 values are int8, sign-extended --, EPID_I32 for bpp 4,
 * EPID_I64 for bpp 8), or EPID_U16: the reference's values checked against [0, 65535] (EPID_XIM_U16_RANGE, never wrapped).
 * status[f] (host, int32 [n]): EPID_XIM_*.  The frames of a failed status hold unspecified values.  h >= 2 (the reference raises
 * ValueError for one row); bpp outside {1, 2, 4, 8} returns EPID_ERR_INVALID (ValueError, like the reference). */
enum {
    EPID_XIM_OK = 0,
    EPID_XIM_LOOKUP_CODE3 = 1,     /* a 2-bit code 3 anywhere in the lookup table: KeyError (LOOKUP_CONVERSION[3]) */
    EPID_XIM_SHORT_BUFFER = 2,     /* the pixel buffer holds fewer bytes than the raw head + the coded diffs: ValueError */
    EPID_XIM_U16_RANGE = 3         /* EPID_U16 output: a value outside [0, 65535]: ValueError (like image.frame_u16) */
};
int32_t epid_xim_decode(epid_ctx* ctx, const void* arena, size_t arena_bytes, const int64_t* desc, int32_t n, int32_t h, int32_t w,
                        int32_t bpp, int32_t dtype, int32_t* status, epid_batch** out);

/* ----------------------------------------------------------------------------------------- machine-log fluence
 * FluenceBase.calc_map(resolution, equal_aspect) (log_analyzer.py:478-612) for a batch of n trajectory logs / Dynalogs, actual
 * (kinds bit 0) and expected (bit 1) in one launch sequence.  `arena` (host, page-locked for a DMA copy) holds every log's column
 * table; logs: n descriptors of 88 bytes (pylinac_b200/log_analyzer.py LOG_DESC_DTYPE, csrc/logs.cu LogDesc): byte offset,
 * snapshot / column strides, element size (float32 trajectory-log body or float64 Dynalog columns), the MU / jaw X1 / X2 / leaf
 * columns, the slice of `snaps` holding the beam-on snapshot indices, the slice of `pair_flags` (bit 0: pair under a Y jaw,
 * MLC.leaf_under_y_jaw :1260-1290; bit 1: pair moved, MLC.pair_moved :1002-1016), the slice of `rows` ([start, stop) output
 * rows per pair, from the reference's int cast of the leaf-width cumsum) and per kind bit 0 "map stays zero" (no beam-on
 * snapshot, max(MU) < 0.5) and bit 1 "divide by MU_total" (MU_total == 25000, :608-610).  out_*: float64 batches [n][h][w]
 * (w = int(400 / resolution)); a kind not requested is returned as NULL.  Bit-identical to the reference: float32 line, double
 * rounding per snapshot, round-half-even edges, numpy slice semantics. */
int32_t epid_log_fluence(epid_ctx* ctx, const void* arena, size_t arena_bytes, const void* logs, int32_t n, const int32_t* snaps,
                         int32_t n_snaps, const uint8_t* pair_flags, int32_t n_pair_flags, const int32_t* rows, int32_t n_rows,
                         double resolution, int32_t w, int32_t h, int32_t kinds, epid_batch** out_actual, epid_batch** out_expected);
/* BaseImage.check_inversion_by_histogram() (core/image.py:899-926) of float64 frames: np.percentile(a, 5 / 50 / 95) from exact order
 * statistics (radix select), and where |p50 - p5| > |p50 - p95| the frame is inverted (-a + max + min, core/array_utils.py:75-77).
 * out: a new float64 batch; inverted (host, int32 [n], may be NULL): the per-frame decision.  Frames must hold no nan. */
int32_t epid_hist_invert(epid_ctx* ctx, const epid_batch* in, epid_batch** out, int32_t* inverted);
/* GammaFluence.calc_map statistics (log_analyzer.py:743-748) per frame of a float64 gamma batch: sum and count of the non-nan
 * values and the count below 1 (host: avg_gamma = sum / count or 0, pass_prcnt = passing / count * 100).  Outputs are host arrays [n]. */
int32_t epid_gamma_stats(epid_ctx* ctx, const epid_batch* gamma, double* sum, int64_t* count, int64_t* passing);

/* ----------------------------------------------------------------------------------------- CT stacks (WinstonLutz.from_cbct)
 * epid_stack_mip: the two maximum-intensity projections of winston_lutz.py:1465-1489 for a volume [N][H][W] of slices in sorted
 * order (I16 or U16; other dtypes EPID_ERR_UNSUPPORTED, as are slices wider than 2048 pixels): np.stack(images, axis=-1).max(axis=0)
 * -> colmax, a new batch [W][1][N], and .max(axis=1) -> rowmax [H][1][N], in the volume's dtype.  Each row is one 1-D signal, the
 * layout epid_zoom takes to resample the slice axis.  One read of the volume; integer max, exact.
 * epid_cbct_views: the four pseudo-cardinal frames of winston_lutz.py:1470-1505 from zoomed projections (epid_zoom output, float64
 * [P][1][N']): for z0 (then z1, which may be NULL and must have z0's shape) frame 2 p = np.rot90(z, 1) and frame 2 p + 1 = its
 * np.fliplr.  Values are rounded like scipy.ndimage.zoom's integer output of src_dtype (I16: half away from zero; U16: + 0.5; both
 * clamped to the type) and stored as the 16 bits array_to_dicom writes (PixelRepresentation 0: int16 bits read back as uint16).
 * out: a new U16 batch [2 or 4][N'][P]. */
int32_t epid_stack_mip(epid_ctx* ctx, const epid_batch* volume, epid_batch** colmax, epid_batch** rowmax);
int32_t epid_cbct_views(epid_ctx* ctx, const epid_batch* z0, const epid_batch* z1, int32_t src_dtype, epid_batch** out);

/* ----------------------------------------------------------------------------------------- light / radiation field coincidence
 * StandardImagingFC2 and its subclasses (IMTLRad, DoselabRLf, IsoAlign, SNCFSQA; planar_imaging.py:1169-1727) and
 * QuasarLightRadScaling (contrib/quasar.py:1-66) for a batch of uint16 frames, one result per frame:
 *   ImagePhantomBase.__init__ ground / normalize (:226-231), check_inversion (core/image.py:868-897), invert, _find_field_info
 *   (strip means -> FWXMProfilePhysical(ground, BEAM_CENTER)), _determine_bb_set, _detect_bb_centers (median filter, near-edge
 *   equalize_adapthist + median filter, SizedDiskLocator.from_center_physical per BB), Quasar's _detect_scaling_centers.
 * The set of nominal BB positions comes from the host (bb_mm: nbb (x, y) pairs; bb15_mm: the 15x15 set of set_mode 1).  Averages,
 * offsets and the SNC FSQA virtual centre are host arithmetic on the returned points. */
#define EPID_LR_MAX_BB 5
#define EPID_LR_SCALING 5
enum {
    EPID_LR_OK = 0,
    EPID_LR_NO_FIELD = 1,     /* no FWXM peak in a strip profile: IndexError in FWXMProfile.field_edge_idx */
    EPID_LR_MISMATCH = 2,     /* x and y field widths differ by more than 10 mm (FC-2 set selection): ValueError */
    EPID_LR_NO_BB = 3,        /* a BB window (or the Quasar scaling window) holds fewer disks than required: ValueError */
    EPID_LR_CAPACITY = 4      /* a search window or region larger than the locator's shared-memory tiles */
};
enum { EPID_LR_SET_FIXED = 0, EPID_LR_SET_FC2 = 1, EPID_LR_SET_QUASAR = 2 };
typedef struct {
    double dpmm;
    double fwxm;                       /* percent */
    double bb_edge_threshold_mm;
    double bb_size_mm, bb_box_mm, strip_width_mm;
    double quasar_offset_mm;           /* set_mode EPID_LR_SET_QUASAR: BBs this far inside the field corners */
    double bb_mm[2 * EPID_LR_MAX_BB], bb15_mm[2 * EPID_LR_MAX_BB];
    int32_t nbb, set_mode;
    int32_t normalize, invert;
    int32_t clahe_kernel;              /* int(round(bb_size_mm / 2 * dpmm * kernel_size_multiplier)) */
    int32_t scaling;                   /* Quasar: locate the 5 scaling BBs in a 35 mm window about the image centre */
} epid_lr_params;

typedef struct { /* one per frame */
    int32_t status;
    int32_t inverted;                  /* check_inversion fired (before the `invert` argument is applied) */
    int32_t large_set;                 /* set_mode EPID_LR_SET_FC2: the 15x15 positions were used */
    int32_t near_edge_mask;            /* bit k: BB k was located on the equalised (CLAHE) image */
    int32_t failed_bb;                 /* EPID_LR_NO_BB: index of the first BB that was not found (nbb: the scaling search) */
    int32_t n_found;                   /* disks found in that window */
    int32_t n_scaling;
    int32_t pad;
    double field_center_x, field_center_y, field_width_x_mm, field_width_y_mm;
    double bb_x[EPID_LR_MAX_BB], bb_y[EPID_LR_MAX_BB];
    double scaling_x[EPID_LR_SCALING], scaling_y[EPID_LR_SCALING];
} epid_lr_result;

int32_t epid_lightrad_analyze(epid_ctx* ctx, const epid_batch* frames, const epid_lr_params* p, epid_lr_result* results);

/* Diagnostic read-back of the light / rad stages: the launch sequence of epid_lightrad_analyze (same results), and per frame the
 * host uint16 [n][h][w] planes of the first 3 x 3 median of the mapped frame (filtered), the equalize_adapthist output before the
 * second median (equalised) and the second median (equalised_filtered), plus EPID_LR_INFO int64 values per frame in the order
 * mn, mx, sum, corner, checked, inv, near_mask, fmn, fmx, umin, umax (raw range, raw frame sum, raw sum of the four corner boxes,
 * check_inversion, final inversion, near-edge mask, range of the filtered frame, range of the equalised frame).  For frames with
 * near_mask == 0 the equalised planes and fmn .. umax are unspecified. */
#define EPID_LR_INFO 11
int32_t epid_lightrad_stages(epid_ctx* ctx, const epid_batch* frames, const epid_lr_params* p, epid_lr_result* results,
                             uint16_t* filtered, uint16_t* equalised, uint16_t* equalised_filtered, int64_t* info);

/* ----------------------------------------------------------------------------------------- nuclear medicine
 * pylinac.nuclear.PlanarUniformity (nuclear.py:151-500): NEMA integral and differential uniformity of uint16 gamma-camera flood frames,
 * bit-identical to the reference.  Per frame: bin x bin block sums (zero-padded bottom / right), the 9-point filter as the integer
 * S = 16 x filtered value with the outer rows / columns zeroed, the threshold (mean of the values above 10 % of the max, times
 * `threshold`), the stray-pixel stencil, the largest 4-connected component (lowest label on ties) and its longest bounding-box side L,
 * erosion k = rint(erode[k] * L) with erode = 1 - size computed by the caller, FOV k = exact EDT > erosion / 2, and the uniformities of
 * the non-zero FOV pixels.  Index 0 of every pair is the UFOV, 1 the CFOV; du_* are indexed [2 * fov + axis], axis 0 being windows of
 * `window` pixels down a column.  The row is a plain struct (not a typedef): its layout is checked by tests/test_nuclear_host.py. */
enum { EPID_NM_OK = 0, EPID_NM_NO_COMPONENT = 1 /* no foreground pixel survives the cleaning (get_fov raises) */ };
struct epid_nm_result { /* one per frame */
    int32_t status;
    int32_t longest;                   /* L */
    int32_t erosion[2];
    int32_t n_fov[2];                  /* non-zero FOV pixels (0: integral_uniformity raises) */
    int32_t max_index[2];              /* first raster index (row * wb + col) of the FOV maximum / minimum */
    int32_t min_index[2];
    int32_t du_count[4];               /* windows holding a FOV pixel (0: differential_uniformity raises) */
    int32_t du_index[4];               /* first (i, j) in row-major order of du_max, as i * wb + j */
    double threshold;                  /* the absolute threshold on S / 16 (nan for a blank frame) */
    double iu[2];                      /* integral uniformity, % */
    double du_max[4];                  /* maximum window uniformity, % */
};

/* frames: uint16 batch; bin: a power of two up to 64; window >= 1.  results: host rows [n].  cleaned (may be NULL): a new float64
 * batch [n][hb][wb] of S / 16 (the reference's binned_frame); masks (may be NULL): a new uint8 batch [2n][hb][wb], the UFOV and CFOV
 * masks of frame k at 2k and 2k + 1.  Non-uint16 frames or bins return EPID_ERR_UNSUPPORTED. */
int32_t epid_nm_uniformity(epid_ctx* ctx, const epid_batch* frames, int32_t bin, double ufov_erode, double cfov_erode, int32_t window,
                           double threshold, struct epid_nm_result* results, epid_batch** cleaned, epid_batch** masks);
/* Diagnostic read-back: the launch sequence of epid_nm_uniformity and host planes [n][hb][wb] of S after the filter (filtered), S after
 * the threshold and stencil (cleaned) and the squared EDT (edt2, -1 for a frame without a component), plus masks [n][2][hb][wb]. */
int32_t epid_nm_stages(epid_ctx* ctx, const epid_batch* frames, int32_t bin, double ufov_erode, double cfov_erode, int32_t window,
                       double threshold, struct epid_nm_result* results, uint32_t* filtered, uint32_t* cleaned, int32_t* edt2, uint8_t* masks);
/* pylinac.nuclear.get_fov on n binary frames (uint8, non-zero = foreground): status, longest, erosion[0] = rint(erode * L) and n_fov[0]
 * of each row, and mask: a new uint8 batch [2n][h][w] whose frame 2k is the eroded binary of frame k. */
int32_t epid_nm_fov(epid_ctx* ctx, const epid_batch* binary, double erode, struct epid_nm_result* results, epid_batch** mask);

/* pylinac.nuclear.TomographicContrast (nuclear.py:1553-1856) on uint16 SPECT volumes, bit-identical to the reference.  A batch of
 * volumes is a uint16 batch of n = volumes x nz slices, volume v being slices v * nz .. v * nz + nz - 1.  The rows are plain structs
 * (not typedefs): their layouts are checked by tests/test_tomo_contrast_host.py. */
enum { EPID_NT_OK = 0, EPID_NT_NO_COMPONENT = 1 /* no pixel at or above 10 % of the volume's maximum: slice_data skips the slice */ };
struct epid_nt_slice { /* one per slice: slice_data (nuclear.py:1620-1651) before the area filter */
    int32_t status;
    int32_t longest;                   /* longest bounding-box side of the largest 4-connected region (first label on ties) */
    int32_t erosion;                   /* rint(ufov_erode * longest) */
    int32_t area;                      /* pixels of the FOV: exact EDT of the whole binary > erosion / 2 */
    int32_t max, min;                  /* of the FOV pixels (0 when the FOV is empty) */
    uint64_t sum;                      /* exact sum of the FOV pixels */
    double centroid_row;               /* the largest region's centroid: exact coordinate sum / area, one rounding */
    double centroid_col;
    double uniformity;                 /* michelson of the FOV pixels (nan for an empty FOV) */
    double value;                      /* their mean (nan for an empty FOV) */
};
struct epid_nt_sphere_in { /* one sphere search: minimize(contrast_f, x0, method="Nelder-Mead", bounds=(lb, ub)) (nuclear.py:1714-1724) */
    double x0[3];                      /* (col, row, z) */
    double lb[3];
    double ub[3];
    double r2;                         /* radius**2 as Python computes it */
    double baseline;                   /* uniformity_value */
    int32_t volume;                    /* index of the volume in the batch */
    int32_t pad;
};
struct epid_nt_sphere { /* the search's result and the sphere at res.x */
    int32_t nfev, nit;
    int32_t status;                    /* scipy's warnflag: 0 converged, 1 maxfun reached, 2 maxiter reached */
    int32_t n_empty;                   /* evaluations whose sphere held no voxel ("Mean of empty slice") */
    int32_t count;                     /* voxels of the sphere at res.x */
    int32_t min;                       /* their minimum (0 when count is 0) */
    uint64_t sum;                      /* their exact sum */
    double x[3];                       /* res.x */
    double fun;                        /* res.fun */
};
/* slice_data's per-slice quantities of every slice (results: host rows [n]); ufov_erode = 1 - ufov_ratio computed by the caller. */
int32_t epid_nt_slices(epid_ctx* ctx, const epid_batch* volumes, int32_t nz, double ufov_erode, struct epid_nt_slice* results);
/* nspheres sphere searches (spheres, results: host rows [nspheres]), each scipy 1.18.1's _minimize_neldermead with its default
 * options, bounds and at most maxfun evaluations and maxiter iterations (minimize() passes 600 for both in 3-D). */
int32_t epid_nt_spheres(epid_ctx* ctx, const epid_batch* volumes, int32_t nz, const struct epid_nt_sphere_in* spheres, int32_t nspheres,
                        int32_t maxfun, int32_t maxiter, struct epid_nt_sphere* results);

/* pylinac.nuclear.TomographicUniformity (nuclear.py:1370-1551) on uint16 SPECT volumes, bit-identical to the reference.  A batch of
 * volumes is a uint16 batch of n = volumes x nz slices, as for epid_nt_slices.  Per volume: the mean m = T / count of the slab of
 * slices first .. first + count - 1 (T the exact integer sum), then epid_nm_uniformity's pipeline on that float64 frame with every sum
 * in numpy's / scipy's order, three FOVs (0 UFOV, 1 CFOV, 2 center; erosion k = rint(erode[k] * L) with erode = 1 - size computed by
 * the caller) and the sums of center_border_ratio.  du_* are indexed [2 * fov + axis].  The row is a plain struct (not a typedef):
 * its layout is checked by tests/test_tomo_uniformity_host.py.  status takes the EPID_NM_* values. */
struct epid_tu_result { /* one per volume */
    int32_t status;
    int32_t longest;                   /* L */
    int32_t erosion[3];
    int32_t n_fov[3];                  /* non-zero FOV pixels (0: integral_uniformity raises) */
    int32_t max_index[3];              /* first raster index (row * wb + col) of the FOV maximum / minimum */
    int32_t min_index[3];
    int32_t du_count[6];               /* windows holding a FOV pixel; the others are all-nan windows */
    int32_t du_index[6];               /* first (i, j) in row-major order of du_max, as i * wb + j */
    int32_t center_count;              /* non-zero pixels of the center FOV */
    int32_t ring_count;                /* non-zero pixels of the UFOV outside the CFOV */
    double threshold;                  /* the absolute threshold (nan when no value exceeds 10 % of the max) */
    double iu[3];                      /* integral uniformity, % */
    double du_max[6];                  /* maximum window uniformity, % */
    double center_sum;                 /* np.sum of the frame, zero outside those pixels */
    double ring_sum;
};
/* bin: a power of two up to 64; window >= 1; 0 <= first, 1 <= count, first + count <= nz.  results: host rows [volumes].  mean,
 * cleaned, masks (each may be NULL): new batches, float64 [volumes][h][w] (the slab mean), float64 [volumes][hb][wb] (the reference's
 * binned_frame) and uint8 [3 x volumes][hb][wb] (the three masks of volume k at 3k .. 3k + 2). */
int32_t epid_tu_uniformity(epid_ctx* ctx, const epid_batch* volumes, int32_t nz, int32_t first, int32_t count, int32_t bin,
                           double ufov_erode, double cfov_erode, double center_erode, int32_t window, double threshold,
                           struct epid_tu_result* results, epid_batch** mean, epid_batch** cleaned, epid_batch** masks);
/* Diagnostic read-back: the launch sequence of epid_tu_uniformity and host planes of the mean [volumes][h][w], the binned, filtered and
 * cleaned frames [volumes][hb][wb], the squared EDT (-1 for a frame without a component) and the masks [volumes][3][hb][wb]. */
int32_t epid_tu_stages(epid_ctx* ctx, const epid_batch* volumes, int32_t nz, int32_t first, int32_t count, int32_t bin,
                       double ufov_erode, double cfov_erode, double center_erode, int32_t window, double threshold,
                       struct epid_tu_result* results, double* mean, double* binned, double* filtered, double* cleaned, int32_t* edt2,
                       uint8_t* masks);

/* CT phantom localization: pylinac.ct's Slice.phantom_roi (ct.py:381-433) with get_regions (ct.py:3315-3348, fill_holes, Otsu
 * threshold), for every listed slice of an int16 or uint16 series, each stage bit-identical to the numpy / scipy / skimage call it
 * restates (DESIGN.md 4.19, 4.20).  Both branches of get_regions: the ndarray branch (clip_in_localization, the cheese phantoms) and
 * the Slice branch (CatPhanBase's default, ct.py:403-406 and 3326-3340: Otsu over skimage.draw.disk(image centre, 110 mm) times 0.8,
 * no clipping).  The rows are plain structs (not typedefs): their layouts are checked by tests/test_cheese_host.py and
 * tests/test_acr_host.py. */
enum {
    EPID_CT_OK = 0,
    EPID_CT_NO_EDGES = 1,     /* max(scharr(HU)) < 0.1: "No edges were found ..." */
    EPID_CT_NO_REGIONS = 2,   /* no region left after thresholding: "The number of ROIs detected ..." */
    EPID_CT_WRONG_SIZE = 3    /* the closest region is more than 1.3x off catphan_size: "Unable to find ROI of expected size ..." */
};
struct epid_ct_slice { /* one per listed slice */
    int32_t status;
    int32_t n_regions;                 /* regions after the fill (0 when the edge check fails) */
    int32_t label;                     /* raster index (row * w + col) of the chosen region's first pixel, -1 if none */
    int32_t area;                      /* its area (= filled_area) */
    double centroid_row;               /* coords.mean(axis=0) of its pixels (nan if none) */
    double centroid_col;
    double max_edge;                   /* max(scharr(HU)) */
    double threshold;                  /* threshold_otsu of the smoothed edges (times 0.8 on the Slice branch) */
};
/* ct.py:381-433 Slice.phantom_roi for every listed slice.  slope / intercept: per slice of the whole series (index = slice); slices
 * [nslices]: the slices to localize, results [nslices] on the host.  catphan_size: the expected area in px^2.  gauss_w
 * [2 gauss_r + 1]: gaussian_filter1d's reversed weights for sigma 1 (mode 'nearest').  otsu_disk_radius > 0 (at least 1 pixel)
 * selects the Slice branch, which requires clip_in_localization 0; otsu_disk_radius <= 0 the ndarray branch, which requires
 * clip_in_localization 1.  clip_in_localization 0 without a disk returns EPID_ERR_UNSUPPORTED, a disk with clipping EPID_ERR_INVALID.
 * scharr, smoothed (float64), filled (uint8) and labels (int32: the union-find root of each pixel of the final mask as an index within
 * its slice, -1 off it), each may be NULL: host planes [nslices][h][w] of the Scharr edges the Gaussian smooths (of the clipped HU on
 * the ndarray branch, of the HU on the Slice branch), the smoothed edges, the mask after binary_fill_holes and its labels. */
int32_t epid_ct_localize(epid_ctx* ctx, const epid_batch* volume, const double* slope, const double* intercept, const int32_t* slices,
                         int32_t nslices, double catphan_size, int32_t clear_borders, int32_t clip_in_localization,
                         double otsu_disk_radius, const double* gauss_w, int32_t gauss_r, struct epid_ct_slice* results,
                         double* scharr, double* smoothed, uint8_t* filled, int32_t* labels);

struct epid_ct_region { /* one per region of get_regions(slice), in skimage's label order */
    int32_t label;                     /* skimage's label: 1 + the region's rank in raster order of first pixels */
    int32_t first;                     /* raster index (row * w + col) of the region's first pixel */
    int32_t area;
    int32_t filled_area;               /* binary_fill_holes of the region's own bbox crop (4-connected background) */
    int32_t bbox[4];                   /* min_row, min_col, max_row + 1, max_col + 1, as skimage's bbox */
    uint64_t sum_r;                    /* exact sums of the pixels' rows and columns: centroid = sum / area */
    uint64_t sum_c;
    uint64_t m_rr;                     /* exact second moments about the bbox corner: sum (r - min_row)^2, sum (c - min_col)^2, */
    uint64_t m_cc;                     /* sum (r - min_row) (c - min_col) */
    uint64_t m_rc;
};
/* ct.py:3315-3348 get_regions(slice) with its defaults, as CatPhanBase.find_phantom_roll (ct.py:2541) calls it, for one slice: the
 * Slice branch's Scharr, Gaussian and disk Otsu times 0.8 (otsu_disk_radius > 0, at least 1 pixel), clear_border, no hole filling,
 * 8-connected labels.  regions [capacity] on the host gets the first min(count, capacity) rows; *count the number of regions,
 * *threshold the slice's threshold and *max_edge max(scharr(HU)).  The other arguments are epid_ct_localize's. */
int32_t epid_ct_regions(epid_ctx* ctx, const epid_batch* volume, const double* slope, const double* intercept, int32_t slice,
                        double otsu_disk_radius, const double* gauss_w, int32_t gauss_r, struct epid_ct_region* regions,
                        int32_t capacity, int32_t* count, double* threshold, double* max_edge);

/* ----------------------------------------------------------------------------------------- multi-GPU (NCCL)
 * The batch shards by frame index with no data-path collective; the only exchange is the final gather of the
 * fixed-size per-frame result structs (SURVEY.md 8e).  id: 128-byte ncclUniqueId created by rank 0. */
int32_t epid_comm_unique_id(void* id128);
int32_t epid_comm_init(epid_ctx* ctx, int32_t nranks, int32_t rank, const void* id128);
int32_t epid_comm_destroy(epid_ctx* ctx);
/* size and rank of ctx's communicator (1, 0 until epid_comm_init succeeded): lets the host side check that the gather it is about
 * to post matches the job's world size instead of silently taking the single-rank path */
int32_t epid_comm_info(const epid_ctx* ctx, int32_t* nranks, int32_t* rank);
/* all ranks contribute bytes_per_rank bytes (host); `all` (host, nranks*bytes_per_rank) is filled on every rank */
int32_t epid_gather_results(epid_ctx* ctx, const void* local, size_t bytes_per_rank, void* all);
int32_t epid_barrier(epid_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* EPID_H */
