// ukf_rtc.cu — UKF and CKF instances around USER-SUPPLIED process / measurement functions.
//
// The reference takes fx(x, dt, **args) and hx(x, **args) as Python callables (filterpy/kalman/UKF.py:
// 284-288, called at :521-522 and :463-464).  A device cannot call back into Python, so the drop-in
// takes them as CUDA C++ source text instead: bke_ukf_model_compile() wraps the text around the very
// kernel the pre-built instances use (ukf_kernel.cuh, model ids BKE_FX_USER / BKE_HX_USER), compiles it
// for sm_90a with NVRTC (libnvrtc is dlopen'ed: libbke.so does not link it), loads the cubin with
// cudaLibraryLoadData and launches the resulting cudaKernel_t like any other kernel.  No CPU path.
// bke_ckf_model_compile does the same around the cubature kernel (ckf_kernel.cuh, CubatureKalmanFilter.py:
// 314-321, 354-363), and bke_enkf_model_compile around the ensemble kernel (enkf_kernel.cuh,
// ensemble_kalman_filter.py:250-251, 279-280); the handle records its family and each step entry point
// refuses the others'.
//
// Program text handed to NVRTC (the user's part between the markers):
//     typedef double real;                       // or float
//     #define BKE_DIM_X 6 / BKE_DIM_Z 3
//     #include "ukf_kernel.cuh"                  // (UKF: also ukf_rts_kernel.cuh)
//     /* user */ __device__ void fx(const real *x, real *out, real dt, const real *args) { ... }
//     /* user */ __device__ void hx(const real *x, real *z, const real *args) { ... }
//     template <> bke_user_fx<real> -> ::fx, bke_user_hx<real> -> ::hx
// A UKF handle's measurement scores (bke_ukf_score_model) are compiled on the first call, as a program of their own: the
// same text with ukf_score_kernel.cuh included and the score kernel as its one name.  Compiling them with the step would
// add a quarter or more to every handle's compile time, whether it ever scores or not.
#include <dlfcn.h>
#include <mutex>
#include <nvrtc.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include "sigma_launch.cuh"
#include "ukf_rts_launch.cuh"

// the filter family a compiled model's kernels belong to
enum { BKE_FAMILY_UKF = 0, BKE_FAMILY_CKF = 1, BKE_FAMILY_ENKF = 2 };

struct bke_ukf_model {
    int family;
    int n, m, dtype, fx_model, hx_model;
    cudaLibrary_t lib;
    cudaKernel_t kern[2];          // [0] plain, [1] with the optional outputs
    cudaKernel_t kern_rts;         // RTS smoother around the user's fx or hooks (NULL: neither, or dim_x > UR_MAXN)
    cudaLibrary_t score_lib;       // UKF: the measurement scores (bke_ukf_score_model), compiled on its first call
    cudaKernel_t kern_score;
    std::string source, include_dirs;   // what the score program is compiled from
    unsigned hooks;                // BKE_HOOK_* mask the program was compiled with
    bool simplex;                  // UKF: compiled for the simplex point set (BKE_UKF_SIMPLEX)
    int regs[2];
    std::string log;
};

namespace bke {
namespace {

struct Nvrtc {
    void *h = nullptr;
    decltype(&nvrtcCreateProgram) create;
    decltype(&nvrtcCompileProgram) compile;
    decltype(&nvrtcDestroyProgram) destroy;
    decltype(&nvrtcGetProgramLogSize) log_size;
    decltype(&nvrtcGetProgramLog) log;
    decltype(&nvrtcGetCUBINSize) cubin_size;
    decltype(&nvrtcGetCUBIN) cubin;
    decltype(&nvrtcAddNameExpression) add_name;
    decltype(&nvrtcGetLoweredName) lowered;
    decltype(&nvrtcGetErrorString) errstr;
};

// libnvrtc: BKE_NVRTC_LIB (set by the Python loader to the copy next to torch's CUDA libraries), the
// loader path, then the toolkit directory
Nvrtc *nvrtc()
{
    static Nvrtc n;
    static bool tried = false;
    if (tried) return n.h ? &n : nullptr;
    tried = true;
    std::vector<std::string> cand;
    if (const char *e = getenv("BKE_NVRTC_LIB")) cand.push_back(e);
    cand.push_back("libnvrtc.so.12");
    cand.push_back("/usr/local/cuda/lib64/libnvrtc.so.12");
    cand.push_back("libnvrtc.so");
    for (const auto &c : cand) {
        n.h = dlopen(c.c_str(), RTLD_NOW | RTLD_LOCAL);
        if (n.h) break;
    }
    if (!n.h) return nullptr;
#define BKE_SYM(field, name) n.field = (decltype(n.field))dlsym(n.h, #name); if (!n.field) { n.h = nullptr; return nullptr; }
    BKE_SYM(create, nvrtcCreateProgram) BKE_SYM(compile, nvrtcCompileProgram) BKE_SYM(destroy, nvrtcDestroyProgram)
    BKE_SYM(log_size, nvrtcGetProgramLogSize) BKE_SYM(log, nvrtcGetProgramLog) BKE_SYM(cubin_size, nvrtcGetCUBINSize)
    BKE_SYM(cubin, nvrtcGetCUBIN) BKE_SYM(add_name, nvrtcAddNameExpression) BKE_SYM(lowered, nvrtcGetLoweredName)
    BKE_SYM(errstr, nvrtcGetErrorString)
#undef BKE_SYM
    return &n;
}

std::string kernel_name(const bke_ukf_model &m, int occ, bool extras)
{
    char buf[256];
    if (m.family == BKE_FAMILY_ENKF) {        // no occupancy parameter: one warp per filter
        snprintf(buf, sizeof buf, "bke::enkfk::enkf_kernel<real, %d, %d, %d, %d, %s>", m.n, m.m, m.fx_model, m.hx_model,
                 extras ? "true" : "false");
        return buf;
    }
    snprintf(buf, sizeof buf, "%s<real, %d, %d, %d, %d, %d, %s%s>", m.family == BKE_FAMILY_CKF ? "bke::ckfk::ckf_kernel" : "bke::ukfk::ukf_kernel",
             m.n, m.m, m.fx_model, m.hx_model, occ, extras ? "true" : "false", m.simplex ? ", true" : "");
    return buf;
}

template <typename T>
int launch_model(const bke_ukf_args &a, const bke_ukf_model &m, const void *fx_args, int64_t s_fx, const void *hx_args, int64_t s_hx,
                 cudaStream_t s)
{
    ukfk::UkfP<T> p;
    ukf_fill_params<T>(a, m.n, p);
    set_user_args<T>(p, fx_args, s_fx, hx_args, s_hx);
    const size_t smem = ukf_smem_bytes<T>(m.n, m.m, m.simplex ? m.n + 1 : 2 * m.n + 1, m.fx_model == BKE_FX_LINEAR, a.F_stride == 0,
                                          m.hx_model == BKE_HX_LINEAR, a.H_stride == 0);
    return launch_kernel((const void *)m.kern[has_extras(a)], ukf_grid(p.N), ukfk::UB, smem, &p, s, "ukf model launch");
}

template <typename T>
int launch_ckf_model(const bke_ckf_args &a, const bke_ukf_model &m, const void *fx_args, int64_t s_fx, const void *hx_args, int64_t s_hx,
                     cudaStream_t s)
{
    ckfk::CkfP<T> p;
    ckf_fill_params<T>(a, p);
    set_user_args<T>(p, fx_args, s_fx, hx_args, s_hx);
    const size_t smem = ukf_smem_bytes<T>(m.n, m.m, 2 * m.n, m.fx_model == BKE_FX_LINEAR, a.F_stride == 0, m.hx_model == BKE_HX_LINEAR,
                                          a.H_stride == 0);
    return launch_kernel((const void *)m.kern[has_extras(a)], ukf_grid(p.N), ukfk::UB, smem, &p, s, "ckf model launch");
}

template <typename T>
int launch_enkf_model(const bke_enkf_args &a, const bke_ukf_model &m, const void *fx_args, int64_t s_fx, const void *hx_args, int64_t s_hx,
                      cudaStream_t s)
{
    enkfk::EnkfP<T> p;
    enkf_fill_params<T>(a, p);
    set_user_args<T>(p, fx_args, s_fx, hx_args, s_hx);
    const size_t smem = enkf_smem_bytes(m.n, a.n_members, sizeof(T));
    return launch_kernel((const void *)m.kern[enkf_has_extras(a)], enkf_grid(p.N), enkfk::EB, smem, &p, s, "enkf model launch");
}

// a *_model step refuses a handle compiled for another family, naming the one it was compiled for
int check_family(const bke_ukf_model &m, int family, const char *fn)
{
    static const char *const name[] = {"UKF (bke_ukf_model_compile)", "CKF (bke_ckf_model_compile)", "EnKF (bke_enkf_model_compile)"};
    if (m.family == family) return BKE_OK;
    set_error("%s: the model was compiled for the %s", fn, name[m.family]);
    return BKE_ERR_BAD_ARG;
}

// the compiled model's shape, element type and models against the step's args
template <typename Args>
int check_match(const Args &a, const bke_ukf_model &m, const char *fn)
{
    if (a.dim_x == m.n && a.dim_z == m.m && a.dtype == m.dtype && a.fx_model == m.fx_model && a.hx_model == m.hx_model) return BKE_OK;
    set_error("%s: args (dim_x=%d dim_z=%d dtype=%d fx=%d hx=%d) do not match the compiled model (%d %d %d %d %d)", fn, a.dim_x, a.dim_z,
              a.dtype, a.fx_model, a.hx_model, m.n, m.m, m.dtype, m.fx_model, m.hx_model);
    return BKE_ERR_BAD_ARG;
}

}  // namespace
}  // namespace bke

using namespace bke;

extern "C" {

// NVRTC half of bke_ukf_model_compile / bke_ckf_model_compile (needs no GPU): program text -> sm_90a cubin
// + the lowered names of the kernel instances of the family (the step with / without the optional outputs and,
// for a UKF around a user fx or hooks, the RTS smoother); `score`: the UKF's measurement-score program instead, whose
// one name is lowered[3]
static int compile_cubin(int family, int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, unsigned hooks,
                         bool simplex, const char *source, const char *include_dirs, std::vector<char> &cubin, std::string (&lowered)[4],
                         std::string &log, bool score = false)
{
    const bool ckf = family == BKE_FAMILY_CKF, enkf = family == BKE_FAMILY_ENKF;
    const char *fn = simplex ? "bke_ukf_model_compile_points"
                   : hooks ? (ckf ? "bke_ckf_model_compile_hooks" : "bke_ukf_model_compile_hooks")
                           : enkf ? "bke_enkf_model_compile" : ckf ? "bke_ckf_model_compile" : "bke_ukf_model_compile";
    if (dim_x < 1 || dim_x > 16 || dim_z < 1 || dim_z > dim_x + 8) { set_error("%s: 1 <= dim_x <= 16, 1 <= dim_z", fn); return BKE_ERR_BAD_ARG; }
    if (int rc = check_dtype(dtype)) return rc;
    const bool ufx = fx_model == BKE_FX_USER, uhx = hx_model == BKE_HX_USER;
    const unsigned all_hooks = BKE_HOOK_X_MEAN | BKE_HOOK_Z_MEAN | BKE_HOOK_RESIDUAL_X | BKE_HOOK_RESIDUAL_Z | BKE_HOOK_STATE_ADD;
    if (hooks) {
        if ((hooks & ~all_hooks) || enkf) { set_error("%s: unknown hook bits 0x%x", fn, hooks); return BKE_ERR_BAD_ARG; }
        if (ckf && hooks != BKE_HOOK_RESIDUAL_Z) {
            set_error("%s: the CKF calls residual_z only (CubatureKalmanFilter.py:376); hooks must be BKE_HOOK_RESIDUAL_Z", fn);
            return BKE_ERR_BAD_ARG;
        }
        if (dim_x > UR_MAXN) { set_error("%s: hooks are supported up to dim_x = %d (got %d)", fn, UR_MAXN, dim_x); return BKE_ERR_UNSUPPORTED; }
        // any model may go with hooks: the built-in transcendental ones read the positions at 0, 2 (, 4)
        if ((!ufx && fx_model != BKE_FX_LINEAR && fx_model != BKE_FX_CONST_VEL) ||
            (!uhx && hx_model != BKE_HX_LINEAR && !(hx_model == BKE_HX_RANGE_BEARING && dim_z == 2 && dim_x >= 3) &&
             !(hx_model == BKE_HX_RANGE_AZ_EL && dim_z == 3 && dim_x >= 5))) {
            set_error("%s: unknown fx / hx model, or a range model whose dim_x / dim_z it cannot serve", fn);
            return BKE_ERR_BAD_ARG;
        }
    } else {
        if (!ufx && !uhx) { set_error("%s: neither fx nor hx is BKE_*_USER (use %s)", fn, enkf ? "bke_enkf_step" : ckf ? "bke_ckf_step" : "bke_ukf_step"); return BKE_ERR_BAD_ARG; }
        if ((!ufx && fx_model != BKE_FX_LINEAR && fx_model != BKE_FX_CONST_VEL) || (!uhx && hx_model != BKE_HX_LINEAR)) {
            set_error("%s: the built-in partner of a user function must be BKE_FX_LINEAR / BKE_FX_CONST_VEL / BKE_HX_LINEAR", fn);
            return BKE_ERR_BAD_ARG;
        }
    }
    if (!ufx && fx_model == BKE_FX_CONST_VEL && (dim_x & 1)) { set_error("BKE_FX_CONST_VEL needs an even dim_x"); return BKE_ERR_BAD_ARG; }
    if (!source || !include_dirs) { set_error("source and include_dirs must be non-NULL"); return BKE_ERR_BAD_ARG; }
    Nvrtc *rt = nvrtc();
    if (!rt) { set_error("libnvrtc.so.12 not found (set BKE_NVRTC_LIB)"); return BKE_ERR_UNSUPPORTED; }

    std::string text;
    text += dtype == BKE_F64 ? "typedef double real;\n" : "typedef float real;\n";
    text += "#define BKE_DIM_X " + std::to_string(dim_x) + "\n#define BKE_DIM_Z " + std::to_string(dim_z) + "\n";
    // the text of a Merwe model without hooks defines neither; with hooks both, in this order
    if (hooks)
        text += "#define BKE_UKF_HOOKS " + std::to_string(hooks) + "u\n";
    if (hooks || simplex)
        text += "#define BKE_N_SIGMAS " + std::to_string(ckf ? 2 * dim_x : simplex ? dim_x + 1 : 2 * dim_x + 1) + "\n";
    text += enkf ? "#include \"enkf_kernel.cuh\"\n" : ckf ? "#include \"ckf_kernel.cuh\"\n" : "#include \"ukf_kernel.cuh\"\n#include \"ukf_rts_kernel.cuh\"\n";
    if (score) text += "#include \"ukf_score_kernel.cuh\"\n";
    text += "#line 1 \"user_model.cu\"\n";
    text += source;
    text += "\n#line 1 \"bke_glue.cu\"\nnamespace bke { namespace ukfk {\n";
    if (ufx) text += "template <> __device__ __forceinline__ void bke_user_fx<real>(const real *x, real *out, real dt, const real *args) { ::fx(x, out, dt, args); }\n";
    if (uhx) text += "template <> __device__ __forceinline__ void bke_user_hx<real>(const real *x, real *z, const real *args) { ::hx(x, z, args); }\n";
    if (hooks & BKE_HOOK_X_MEAN) text += "template <> __device__ __forceinline__ void bke_hook_x_mean<real>(const real *s, const real *w, real *o) { ::x_mean_fn(s, w, o); }\n";
    if (hooks & BKE_HOOK_Z_MEAN) text += "template <> __device__ __forceinline__ void bke_hook_z_mean<real>(const real *s, const real *w, real *o) { ::z_mean_fn(s, w, o); }\n";
    if (hooks & BKE_HOOK_RESIDUAL_X) text += "template <> __device__ __forceinline__ void bke_hook_residual_x<real>(const real *a, const real *b, real *o) { ::residual_x(a, b, o); }\n";
    if (hooks & BKE_HOOK_RESIDUAL_Z) text += "template <> __device__ __forceinline__ void bke_hook_residual_z<real>(const real *a, const real *b, real *o) { ::residual_z(a, b, o); }\n";
    if (hooks & BKE_HOOK_STATE_ADD) text += "template <> __device__ __forceinline__ void bke_hook_state_add<real>(const real *a, const real *b, real *o) { ::state_add(a, b, o); }\n";
    text += "} }\n";

    const int occ = enkf ? 0 : ckf ? ckf_occupancy(dim_x, dtype == BKE_F64)
                                   : ukf_occupancy(dim_x, dtype == BKE_F64, simplex, hx_model == BKE_HX_RANGE_AZ_EL || hx_model == BKE_HX_RANGE_BEARING);
    bke_ukf_model tmp;
    tmp.family = family; tmp.n = dim_x; tmp.m = dim_z; tmp.fx_model = fx_model; tmp.hx_model = hx_model; tmp.simplex = simplex;
    nvrtcProgram prog;
    nvrtcResult r = rt->create(&prog, text.c_str(), enkf ? "bke_enkf_user.cu" : ckf ? "bke_ckf_user.cu" : "bke_ukf_user.cu", 0, nullptr, nullptr);
    if (r != NVRTC_SUCCESS) { set_error("nvrtcCreateProgram: %s", rt->errstr(r)); return BKE_ERR_CUDA; }
    std::vector<std::string> opts = {"--gpu-architecture=sm_90a", "-std=c++17", "-lineinfo", "-default-device"};     // (bke.h declares the host C-ABI)
    {
        std::string dirs = include_dirs;
        size_t pos = 0;
        while (pos <= dirs.size()) {
            size_t e = dirs.find(':', pos);
            if (e == std::string::npos) e = dirs.size();
            if (e > pos) opts.push_back("-I" + dirs.substr(pos, e - pos));
            pos = e + 1;
        }
    }
    std::vector<const char *> copts;
    for (auto &o : opts) copts.push_back(o.c_str());
    // the step kernel with / without the optional outputs and, around a user fx or hooks, the RTS smoother; or the
    // measurement scores alone (an empty name: no such kernel in this program)
    const bool with_rts = !score && !ckf && !enkf && (ufx || hooks) && dim_x <= UR_MAXN;
    std::string names[4];
    if (!score) { names[0] = kernel_name(tmp, occ, false); names[1] = kernel_name(tmp, occ, true); }
    if (with_rts) names[2] = std::string("bke::ukf_rts_kernel<real, ") + (ufx ? "true" : "false") + (simplex ? ", true>" : ">");
    if (score)
        names[3] = "bke::ukfk::ukf_score_kernel<real, " + std::to_string(dim_x) + ", " + std::to_string(dim_z) + ", " +
                   std::to_string(hx_model) + ", " + std::to_string(occ) + (simplex ? ", true>" : ", false>");
    for (int i = 0; i < 4; i++)
        if (!names[i].empty()) rt->add_name(prog, names[i].c_str());
    r = rt->compile(prog, (int)copts.size(), copts.data());
    size_t lsz = 0;
    rt->log_size(prog, &lsz);
    log.clear();
    if (lsz > 1) { log.resize(lsz); rt->log(prog, &log[0]); }
    if (r != NVRTC_SUCCESS) {
        set_error("NVRTC could not compile the %s model: %s\n%s", enkf ? "EnKF" : ckf ? "CKF" : "UKF", rt->errstr(r), log.c_str());
        rt->destroy(&prog);
        return BKE_ERR_BAD_ARG;
    }
    size_t csz = 0;
    rt->cubin_size(prog, &csz);
    cubin.resize(csz);
    rt->cubin(prog, cubin.data());
    for (int i = 0; i < 4; i++) {
        lowered[i].clear();
        if (names[i].empty()) continue;
        const char *ln = nullptr;
        if (rt->lowered(prog, names[i].c_str(), &ln) != NVRTC_SUCCESS || !ln) {
            set_error("nvrtcGetLoweredName failed for %s", names[i].c_str());
            rt->destroy(&prog);
            return BKE_ERR_CUDA;
        }
        lowered[i] = ln;
    }
    rt->destroy(&prog);
    return BKE_OK;
}

static int model_compile(int family, int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, unsigned hooks,
                         const char *source, const char *include_dirs, bke_ukf_model **out, bool simplex = false)
{
    if (!out) { set_error("out is NULL"); return BKE_ERR_BAD_ARG; }
    *out = nullptr;
    std::vector<char> cubin;
    std::string lowered[4], log;
    int rc = compile_cubin(family, dim_x, dim_z, dtype, fx_model, hx_model, hooks, simplex, source, include_dirs, cubin, lowered, log);
    if (rc != BKE_OK) return rc;
    bke_ukf_model *m = new bke_ukf_model();
    m->family = family; m->n = dim_x; m->m = dim_z; m->dtype = dtype; m->fx_model = fx_model; m->hx_model = hx_model; m->lib = nullptr; m->log = log;
    m->hooks = hooks;
    m->simplex = simplex;
    m->kern_rts = nullptr;
    m->score_lib = nullptr;
    m->kern_score = nullptr;
    m->source = source;
    m->include_dirs = include_dirs;
    if (check_cuda(cudaLibraryLoadData(&m->lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0), "cudaLibraryLoadData")) { delete m; return BKE_ERR_CUDA; }
    for (int i = 0; i < 2; i++) {
        if (check_cuda(cudaLibraryGetKernel(&m->kern[i], m->lib, lowered[i].c_str()), "cudaLibraryGetKernel")) {
            cudaLibraryUnload(m->lib); delete m;
            return BKE_ERR_CUDA;
        }
        cudaFuncAttributes fa;
        m->regs[i] = cudaFuncGetAttributes(&fa, (const void *)m->kern[i]) == cudaSuccess ? fa.numRegs : -1;
    }
    if (!lowered[2].empty() && check_cuda(cudaLibraryGetKernel(&m->kern_rts, m->lib, lowered[2].c_str()), "cudaLibraryGetKernel (rts)")) {
        cudaLibraryUnload(m->lib); delete m;
        return BKE_ERR_CUDA;
    }
    cudaGetLastError();
    *out = m;
    return BKE_OK;
}

int bke_ukf_model_compile(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, const char *source,
                          const char *include_dirs, bke_ukf_model **out)
{
    return model_compile(BKE_FAMILY_UKF, dim_x, dim_z, dtype, fx_model, hx_model, 0u, source, include_dirs, out);
}

// the point set of a UKF model: 0 (MerweScaledSigmaPoints, as bke_ukf_model_compile[_hooks]) or BKE_UKF_SIMPLEX
static int check_points(uint32_t points)
{
    if (points != 0u && points != BKE_UKF_SIMPLEX) { set_error("bke_ukf_model_compile_points: points must be 0 or BKE_UKF_SIMPLEX"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int bke_ukf_model_compile_points(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, uint32_t hooks,
                                 uint32_t points, const char *source, const char *include_dirs, bke_ukf_model **out)
{
    if (out) *out = nullptr;
    const int rc = check_points(points);
    if (rc) return rc;
    return model_compile(BKE_FAMILY_UKF, dim_x, dim_z, dtype, fx_model, hx_model, hooks, source, include_dirs, out, points != 0u);
}

int bke_enkf_model_compile(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, const char *source,
                           const char *include_dirs, bke_ukf_model **out)
{
    return model_compile(BKE_FAMILY_ENKF, dim_x, dim_z, dtype, fx_model, hx_model, 0u, source, include_dirs, out);
}

int bke_ckf_model_compile(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, const char *source,
                          const char *include_dirs, bke_ukf_model **out)
{
    return model_compile(BKE_FAMILY_CKF, dim_x, dim_z, dtype, fx_model, hx_model, 0u, source, include_dirs, out);
}

int bke_ukf_model_compile_hooks(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, uint32_t hooks,
                                const char *source, const char *include_dirs, bke_ukf_model **out)
{
    return model_compile(BKE_FAMILY_UKF, dim_x, dim_z, dtype, fx_model, hx_model, hooks, source, include_dirs, out);
}

int bke_ckf_model_compile_hooks(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, uint32_t hooks,
                                const char *source, const char *include_dirs, bke_ukf_model **out)
{
    return model_compile(BKE_FAMILY_CKF, dim_x, dim_z, dtype, fx_model, hx_model, hooks, source, include_dirs, out);
}

// the NVRTC half alone (CPU-only check that a model's text compiles for sm_90a): cubin size or 0
static size_t cubin_bytes(int family, int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, unsigned hooks,
                          const char *source, const char *include_dirs, bool simplex = false, bool score = false)
{
    std::vector<char> cubin;
    std::string lowered[4], log;
    if (compile_cubin(family, dim_x, dim_z, dtype, fx_model, hx_model, hooks, simplex, source, include_dirs, cubin, lowered, log, score) != BKE_OK)
        return 0;
    return cubin.size();
}

size_t bke_debug_ukf_model_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, const char *source,
                                       const char *include_dirs)
{
    return cubin_bytes(BKE_FAMILY_UKF, dim_x, dim_z, dtype, fx_model, hx_model, 0u, source, include_dirs);
}

size_t bke_debug_ckf_model_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, const char *source,
                                       const char *include_dirs)
{
    return cubin_bytes(BKE_FAMILY_CKF, dim_x, dim_z, dtype, fx_model, hx_model, 0u, source, include_dirs);
}

size_t bke_debug_enkf_model_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model, const char *source,
                                        const char *include_dirs)
{
    return cubin_bytes(BKE_FAMILY_ENKF, dim_x, dim_z, dtype, fx_model, hx_model, 0u, source, include_dirs);
}

size_t bke_debug_ukf_model_hooks_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                             uint32_t hooks, const char *source, const char *include_dirs)
{
    return cubin_bytes(BKE_FAMILY_UKF, dim_x, dim_z, dtype, fx_model, hx_model, hooks, source, include_dirs);
}

size_t bke_debug_ckf_model_hooks_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                             uint32_t hooks, const char *source, const char *include_dirs)
{
    return cubin_bytes(BKE_FAMILY_CKF, dim_x, dim_z, dtype, fx_model, hx_model, hooks, source, include_dirs);
}

size_t bke_debug_ukf_model_points_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                              uint32_t hooks, uint32_t points, const char *source, const char *include_dirs)
{
    if (check_points(points)) return 0;
    return cubin_bytes(BKE_FAMILY_UKF, dim_x, dim_z, dtype, fx_model, hx_model, hooks, source, include_dirs, points != 0u);
}

size_t bke_debug_ukf_score_model_cubin_bytes(int32_t dim_x, int32_t dim_z, int32_t dtype, int32_t fx_model, int32_t hx_model,
                                              uint32_t hooks, uint32_t points, const char *source, const char *include_dirs)
{
    if (check_points(points)) return 0;
    return cubin_bytes(BKE_FAMILY_UKF, dim_x, dim_z, dtype, fx_model, hx_model, hooks, source, include_dirs, points != 0u, true);
}

const char *bke_ukf_model_log(const bke_ukf_model *m) { return m ? m->log.c_str() : ""; }

int bke_ukf_model_registers(const bke_ukf_model *m, int32_t extras) { return m ? m->regs[extras ? 1 : 0] : -1; }

void bke_ukf_model_free(bke_ukf_model *m)
{
    if (!m) return;
    if (m->lib) cudaLibraryUnload(m->lib);
    if (m->score_lib) cudaLibraryUnload(m->score_lib);
    delete m;
}

int bke_ukf_step_model(const bke_ukf_args *args, const bke_ukf_model *model, const void *fx_args, int64_t fx_args_stride,
                       const void *hx_args, int64_t hx_args_stride, void *stream)
{
    if (!args || !model) { set_error("args / model is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_ukf_args &a = *args;
    int rc;
    if ((rc = check_family(*model, BKE_FAMILY_UKF, "bke_ukf_step_model")) || (rc = check_match(a, *model, "bke_ukf_step_model")) ||
        (rc = validate_ukf(a)))
        return rc;
    if (fx_args_stride < 0 || hx_args_stride < 0) { set_error("negative args stride"); return BKE_ERR_BAD_ARG; }
    const bool spx = (a.flags & BKE_UKF_SIMPLEX) != 0;
    if (spx != model->simplex) {
        set_error("bke_ukf_step_model: the model was compiled for the %s point set, the step asks for the %s set",
                  model->simplex ? "simplex" : "Merwe", spx ? "simplex" : "Merwe");
        return BKE_ERR_BAD_ARG;
    }
    if (a.n_filters == 0) return BKE_OK;
    return a.dtype == BKE_F32 ? launch_model<float>(a, *model, fx_args, fx_args_stride, hx_args, hx_args_stride, (cudaStream_t)stream)
                              : launch_model<double>(a, *model, fx_args, fx_args_stride, hx_args, hx_args_stride, (cudaStream_t)stream);
}

int bke_ukf_rts_smoother_model(const bke_ukf_rts_args *args, const bke_ukf_model *model, const void *fx_args, int64_t fx_args_stride,
                               void *stream)
{
    if (!args || !model) { set_error("args / model is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_ukf_rts_args &a = *args;
    int rc = check_family(*model, BKE_FAMILY_UKF, "bke_ukf_rts_smoother_model");
    if (rc) return rc;
    if (!model->kern_rts) { set_error("bke_ukf_rts_smoother_model: the model has neither a user fx nor hooks (use bke_ukf_rts_smoother) or dim_x > %d", UR_MAXN); return BKE_ERR_UNSUPPORTED; }
    if (a.dim_x != model->n || a.dtype != model->dtype || a.fx_model != model->fx_model) { set_error("bke_ukf_rts_smoother_model: args do not match the compiled model"); return BKE_ERR_BAD_ARG; }
    if (((a.flags & BKE_UKF_SIMPLEX) != 0) != model->simplex) {
        set_error("bke_ukf_rts_smoother_model: the model was compiled for the %s point set, the smoother asks for the %s set",
                  model->simplex ? "simplex" : "Merwe", model->simplex ? "Merwe" : "simplex");
        return BKE_ERR_BAD_ARG;
    }
    // unlike the pre-built smoother, F and the strides are checked for an empty bank too
    if (a.fx_model == BKE_FX_LINEAR && (!a.F || a.F_stride < 0)) { set_error("BKE_FX_LINEAR needs F and F_stride >= 0"); return BKE_ERR_BAD_ARG; }
    if (fx_args_stride < 0 || a.Q_stride < 0) { set_error("negative stride"); return BKE_ERR_BAD_ARG; }
    const int v = validate_ukf_rts(a, model->fx_model == BKE_FX_USER);
    if (v >= 0) return v;
    void *params[1];
    UrP<float> pf; UrP<double> pd;
    if (a.dtype == BKE_F32) { ukf_rts_fill_params<float>(a, pf); pf.fx_args = (const float *)fx_args; pf.s_fx_args = fx_args_stride; params[0] = &pf; }
    else { ukf_rts_fill_params<double>(a, pd); pd.fx_args = (const double *)fx_args; pd.s_fx_args = fx_args_stride; params[0] = &pd; }
    if (check_cuda(cudaLaunchKernel((const void *)model->kern_rts, dim3((unsigned)((a.n_filters + 63) / 64)), dim3(64), params, 0, (cudaStream_t)stream),
                   "ukf rts model launch")) return BKE_ERR_CUDA;
    return BKE_OK;
}

// the handle's measurement-score program, compiled and loaded on the first bke_ukf_score_model call
static int load_score_kernel(bke_ukf_model &m)
{
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    if (m.kern_score) return BKE_OK;
    std::vector<char> cubin;
    std::string lowered[4], log;
    int rc = compile_cubin(m.family, m.n, m.m, m.dtype, m.fx_model, m.hx_model, m.hooks, m.simplex, m.source.c_str(), m.include_dirs.c_str(),
                           cubin, lowered, log, true);
    if (rc != BKE_OK) return rc;
    cudaLibrary_t lib;
    if (check_cuda(cudaLibraryLoadData(&lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0), "cudaLibraryLoadData (score)")) return BKE_ERR_CUDA;
    cudaKernel_t k;
    if (check_cuda(cudaLibraryGetKernel(&k, lib, lowered[3].c_str()), "cudaLibraryGetKernel (score)")) { cudaLibraryUnload(lib); return BKE_ERR_CUDA; }
    m.score_lib = lib;
    m.kern_score = k;
    return BKE_OK;
}

}  // extern "C"

template <typename T>
static int launch_score_model(const bke_ukf_score_args &a, const bke_ukf_model &m, const void *hx_args, int64_t s_hx, cudaStream_t s)
{
    ukfk::UkfScoreP<T> p;
    ukf_score_fill_params<T>(a, p);
    p.hx_args = (const T *)hx_args; p.s_hx_args = s_hx;
    const size_t smem = ukf_score_smem_bytes<T>(m.n, m.m, m.simplex, m.hx_model == BKE_HX_LINEAR, a.H_stride == 0);
    // the slot of S^-1 grows with dim_z^2, so a model that steps may still not fit the score's shared memory
    const size_t smem_max = 227 * 1024;                      // the most one CTA may use on sm_90
    if (smem > smem_max) {
        set_error("bke_ukf_score_model: dim_x=%d dim_z=%d needs %zu B of shared memory per CTA (> %zu)", m.n, m.m, smem, smem_max);
        return BKE_ERR_UNSUPPORTED;
    }
    if (int rc = load_score_kernel(const_cast<bke_ukf_model &>(m))) return rc;
    return launch_kernel((const void *)m.kern_score, ukf_grid(p.N), ukfk::UB, smem, &p, s, "ukf score model launch");
}

extern "C" {

int bke_ukf_score_model(const bke_ukf_score_args *args, const bke_ukf_model *model, const void *hx_args, int64_t hx_args_stride, void *stream)
{
    if (!args || !model) { set_error("args / model is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_ukf_score_args &a = *args;
    int rc;
    if ((rc = check_family(*model, BKE_FAMILY_UKF, "bke_ukf_score_model")) || (rc = validate_ukf_score(a))) return rc;
    if (a.dim_x != model->n || a.dim_z != model->m || a.dtype != model->dtype || a.hx_model != model->hx_model) {
        set_error("bke_ukf_score_model: args (dim_x=%d dim_z=%d dtype=%d hx=%d) do not match the compiled model (%d %d %d %d)", a.dim_x,
                  a.dim_z, a.dtype, a.hx_model, model->n, model->m, model->dtype, model->hx_model);
        return BKE_ERR_BAD_ARG;
    }
    if (((a.flags & BKE_UKF_SIMPLEX) != 0) != model->simplex) {
        set_error("bke_ukf_score_model: the model was compiled for the %s point set, the call asks for the %s set",
                  model->simplex ? "simplex" : "Merwe", model->simplex ? "Merwe" : "simplex");
        return BKE_ERR_BAD_ARG;
    }
    if (hx_args_stride < 0) { set_error("negative args stride"); return BKE_ERR_BAD_ARG; }
    if (a.n_filters == 0 || a.n_candidates == 0) return BKE_OK;
    return a.dtype == BKE_F32 ? launch_score_model<float>(a, *model, hx_args, hx_args_stride, (cudaStream_t)stream)
                              : launch_score_model<double>(a, *model, hx_args, hx_args_stride, (cudaStream_t)stream);
}

int bke_ckf_step_model(const bke_ckf_args *args, const bke_ukf_model *model, const void *fx_args, int64_t fx_args_stride,
                       const void *hx_args, int64_t hx_args_stride, void *stream)
{
    if (!args || !model) { set_error("args / model is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_ckf_args &a = *args;
    int rc;
    if ((rc = check_family(*model, BKE_FAMILY_CKF, "bke_ckf_step_model")) || (rc = check_match(a, *model, "bke_ckf_step_model")) ||
        (rc = validate_ckf(a)))
        return rc;
    if (fx_args_stride < 0 || hx_args_stride < 0) { set_error("negative args stride"); return BKE_ERR_BAD_ARG; }
    if (a.n_filters == 0) return BKE_OK;
    return a.dtype == BKE_F32 ? launch_ckf_model<float>(a, *model, fx_args, fx_args_stride, hx_args, hx_args_stride, (cudaStream_t)stream)
                              : launch_ckf_model<double>(a, *model, fx_args, fx_args_stride, hx_args, hx_args_stride, (cudaStream_t)stream);
}

int bke_enkf_step_model(const bke_enkf_args *args, const bke_ukf_model *model, const void *fx_args, int64_t fx_args_stride,
                        const void *hx_args, int64_t hx_args_stride, void *stream)
{
    if (!args || !model) { set_error("args / model is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_enkf_args &a = *args;
    int rc;
    if ((rc = check_family(*model, BKE_FAMILY_ENKF, "bke_enkf_step_model")) || (rc = check_match(a, *model, "bke_enkf_step_model")) ||
        (rc = validate_enkf(a)))
        return rc;
    if (fx_args_stride < 0 || hx_args_stride < 0) { set_error("negative args stride"); return BKE_ERR_BAD_ARG; }
    if (a.n_filters == 0) return BKE_OK;
    return a.dtype == BKE_F32 ? launch_enkf_model<float>(a, *model, fx_args, fx_args_stride, hx_args, hx_args_stride, (cudaStream_t)stream)
                              : launch_enkf_model<double>(a, *model, fx_args, fx_args_stride, hx_args, hx_args_stride, (cudaStream_t)stream);
}

}  // extern "C"
