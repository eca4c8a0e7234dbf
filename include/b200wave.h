/*
 * b200wave.h -- C ABI of libb200wave.so: the H100 (sm_90a) 2-D wavelet filterbank engine.
 *
 * This is the drop-in boundary for the ONE hot path of fbcotter/pytorch_wavelets:
 * the per-level separable analysis / synthesis filter banks behind DWTForward / DWTInverse,
 * DTCWTForward / DTCWTInverse and the ScatLayer magnitude epilogue.  The reference has no FFI
 * of its own; its narrowest stable interface is the torch.autograd.Function layer, so there is
 * exactly one entry point here per reference Function.forward (each cites the reference
 * file:line it replaces).  INTEGRATION.md shows the ctypes stub a maintainer of the reference
 * would add to bind them.
 *
 * Conventions
 *   - All image tensors are fp32, device memory, NCHW; "planes" = N*C independent images.
 *   - Filter taps are HOST pointers to fp32 arrays holding the taps exactly as the reference
 *     stores them in its module buffers (analysis filters time-reversed, synthesis filters
 *     as-is: reference dwt/lowlevel.py:916-920,970; dtcwt/lowlevel.py:58-67).  They are copied
 *     into kernel parameters (constant bank) by value; no device filter memory is needed.
 *   - The caller owns every buffer, including outputs; the library never allocates device
 *     memory, keeps no reference after return, has no global mutable state and is re-entrant.
 *   - Every call is asynchronous on the given CUDA stream (a cudaStream_t passed as void*;
 *     NULL = legacy default stream) and never synchronises the host.
 *   - Return value: 0 on success, a negative B200W_E* code otherwise (b200w_strerror()).
 *     Shape / mode validation mirrors the reference's Python exceptions; the Python shell
 *     raises the same exception types before calling, so C errors are defensive.
 *   - mode integers are the reference's mode_to_int() codes (dwt/lowlevel.py:274-290).
 */
#ifndef B200WAVE_H
#define B200WAVE_H

#ifdef __cplusplus
extern "C" {
#endif

#define B200W_VERSION 100 /* 0.1.0 */

/* reference dwt/lowlevel.py:274-290 */
enum {
  B200W_MODE_ZERO = 0,
  B200W_MODE_SYMMETRIC = 1,
  B200W_MODE_PERIODIZATION = 2,
  B200W_MODE_CONSTANT = 3, /* rejected by the filter banks, as in the reference */
  B200W_MODE_REFLECT = 4,
  B200W_MODE_REPLICATE = 5, /* rejected, as in the reference */
  B200W_MODE_PERIODIC = 6
};

enum {
  B200W_OK = 0,
  B200W_EMODE = -1,   /* unknown / unsupported padding mode  (reference: ValueError "Unkown pad type") */
  B200W_ESIZE = -2,   /* bad tensor size (reference: ValueError rows/cols multiple of 2 or 4)          */
  B200W_EARG = -3,    /* null pointer / inconsistent arguments                                        */
  B200W_EFILTER = -4, /* unsupported filter length                                                   */
  B200W_ECUDA = -5,   /* CUDA launch error (cudaGetLastError captured)                                */
  B200W_ENOTIMPL = -6 /* reference raises NotImplementedError here                                   */
};

#define B200W_MAX_TAPS 40 /* longest supported filter (db20) */

int b200w_version(void);
const char* b200w_strerror(int code);
/* last CUDA error string seen by this thread's most recent failing call ("" if none) */
const char* b200w_last_cuda_error(void);

/* pywt.dwt_coeff_len as used at reference dwt/lowlevel.py:153: ceil(n/2) for periodization,
 * floor((n+flen-1)/2) otherwise.  Returns <0 on bad input. */
int b200w_dwt_coeff_len(int n, int flen, int mode);
/* length produced by one synthesis level from k coefficients (reference dwt/lowlevel.py:242-267):
 * 2k for periodization else 2k - flen + 2. */
int b200w_dwt_rec_len(int k, int flen, int mode);

/* ---------------------------------------------------------------------------------------------
 * K1  one 2-D DWT analysis level.           Replaces AFB2D.forward, reference dwt/lowlevel.py:336-347
 *     (afb1d along W then along H, :91-172; boundary index generation mypad :28-88).
 *   x      (planes, H, W), row pitch x_pitch elements, plane stride x_plane_stride elements
 *   ll     (planes, Ho, Wo) with ll_pitch / ll_plane_stride (lets the caller keep padded internal levels)
 *   highs  (planes, 3, Ho, Wo) contiguous: [lh, hl, hh]; lh = low along W, high along H
 *   fw_*   taps applied along W (the module buffers named *_col -- reference quirk,
 *          dwt/transform2d.py:70-71 vs lowlevel.py:336), length Lw;  fh_* along H, length Lh.
 *   Ho = b200w_dwt_coeff_len(H, Lh, mode), Wo = b200w_dwt_coeff_len(W, Lw, mode).
 * Also computes SFB2D.backward (dwt/lowlevel.py:683-694) when given the synthesis taps.
 */
int b200w_dwt_afb2d(const float* x, long long x_plane_stride, int x_pitch,
                    float* ll, long long ll_plane_stride, int ll_pitch,
                    float* highs,
                    int planes, int H, int W,
                    const float* fw_lo, const float* fw_hi, int Lw,
                    const float* fh_lo, const float* fh_hi, int Lh,
                    int mode, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K1xJ  all J analysis levels in one call.  Replaces the level loop of DWTForward.forward, reference
 *     dwt/transform2d.py:68-74 (J x AFB2D.apply with the low-pass fed back).
 *   x      (planes, H, W) pitched as in K1
 *   yl     (planes, H_J, W_J) contiguous: the final low-pass
 *   highs  HOST array of J device pointers; highs[j] is level j+1's (planes, 3, H_j, W_j) contiguous tensor
 *          (finest first, the reference's yh list); H_j = b200w_dwt_coeff_len(H_{j-1}, Lh, mode) etc.
 *   When the fused pyramid kernel applies (equal even filter lengths <= 16, mode zero / symmetric / reflect,
 *   16-byte aligned rows with W % 4 == 0, every level at least as large as the filter, the plan fits shared
 *   memory) this is ONE kernel launch and the inter-level low-passes never touch device memory.  Otherwise the
 *   levels run one K1 launch each and their intermediate low-passes live in `workspace` (caller-owned device
 *   memory, at least b200w_dwt_forward_workspace(...) bytes, which is 0 when the fused kernel applies; the
 *   same x / strides must be passed to both calls since the answer depends on the alignment of x).
 */
long long b200w_dwt_forward_workspace(const float* x, long long x_plane_stride, int x_pitch,
                                      int planes, int H, int W, int J, int Lw, int Lh, int mode);
int b200w_dwt_forward(const float* x, long long x_plane_stride, int x_pitch,
                      int planes, int H, int W, int J,
                      float* yl, float* const* highs,
                      const float* fw_lo, const float* fw_hi, int Lw,
                      const float* fh_lo, const float* fh_hi, int Lh,
                      int mode, void* workspace, long long workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K2  one 2-D DWT synthesis level.          Replaces SFB2D.forward, reference dwt/lowlevel.py:671-680
 *     (sfb1d along H for (ll,lh) and (hl,hh), then along W; :226-271).
 *   ll     (planes, Hc, Wc) pitched;  highs (planes, 3, Hc, Wc) contiguous, or NULL = zeros
 *          (reference dwt/transform2d.py:137-139)
 *   y      (planes, Ho, Wo) pitched.  Ho/Wo may be smaller than the natural size
 *          b200w_dwt_rec_len(Hc, Lh, mode) -- the crop of AFB2D.backward (lowlevel.py:359-364).
 *   gh_* taps along H (first pass), gw_* along W.
 */
int b200w_dwt_sfb2d(const float* ll, long long ll_plane_stride, int ll_pitch,
                    const float* highs,
                    float* y, long long y_plane_stride, int y_pitch,
                    int planes, int Hc, int Wc, int Ho, int Wo,
                    const float* gh_lo, const float* gh_hi, int Lh,
                    const float* gw_lo, const float* gw_hi, int Lw,
                    int mode, void* stream);

/* ---------------------------------------------------------------------------------------------
 * 1-D DWT levels.                           Replace AFB1D.forward / SFB1D.forward, reference dwt/lowlevel.py:388-404,
 *     717-729 (afb1d / sfb1d along the last dimension; the level loops are DWT1DForward / DWT1DInverse,
 *     dwt/transform1d.py:44-65, 97-115).  Same modes, tap conventions and length rules as K1 / K2.
 *   b200w_dwt_afb1d: x (rows, N) with row pitch x_pitch -> lo, hi (rows, K) contiguous, K = b200w_dwt_coeff_len(N, L, mode)
 *   b200w_dwt_sfb1d: lo, hi (rows, K) contiguous (hi may be NULL = zeros) -> y (rows, Nout) contiguous,
 *                    Nout <= b200w_dwt_rec_len(K, L, mode) (smaller = the crop of AFB1D.backward, :406-424)
 * Each also computes the other's backward pass when given the same stored filters.
 */
int b200w_dwt_afb1d(const float* x, long long x_pitch, int rows, int N, float* lo, float* hi,
                    const float* f0, const float* f1, int L, int mode, void* stream);
int b200w_dwt_sfb1d(const float* lo, const float* hi, int rows, int K, float* y, int Nout,
                    const float* g0, const float* g1, int L, int mode, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Transpose of the mode-extended analysis bank (an addition beyond the reference): the exact adjoint A_m^T of
 * b200w_dwt_afb2d / b200w_dwt_afb1d in every mode, which SFB2D / SFB1D's double backward needs (the reference gets it
 * by differentiating its backward's F.pad / conv2d graph, dwt/lowlevel.py:683-694, 732-743).  It differs from the
 * synthesis bank (K2 cropped to n) in symmetric, reflect, periodic and odd-size periodization mode, where the boundary
 * extension folds the coefficients that reach extended positions back onto the samples they copy.
 *   b200w_dwt_afb2d_adjoint: ll (planes, Hc, Wc) pitched, highs (planes, 3, Hc, Wc) contiguous or NULL = zeros
 *                            -> y (planes, H, W) pitched, with Hc = b200w_dwt_coeff_len(H, Lh, mode) and
 *                            Wc = b200w_dwt_coeff_len(W, Lw, mode).  fh_*: the stored analysis taps of the H pass,
 *                            fw_* of the W pass (b200w_dwt_afb2d's fh / fw).
 *   b200w_dwt_afb1d_adjoint: lo, hi (rows, K) contiguous (hi may be NULL) -> y (rows, N) contiguous,
 *                            K = b200w_dwt_coeff_len(N, L, mode).
 * One call is the synthesis level cropped to the output (the streaming kernels where they apply) followed, outside zero
 * mode and even-size periodization, by one border kernel that rewrites the outputs within L samples of an edge.
 * Errors: B200W_EMODE, B200W_EARG for a NULL required pointer or a pitch below the row length, B200W_ESIZE for a
 * coefficient size that is not the analysis length of the output size, B200W_EFILTER for L < 2 or L > 40.
 */
int b200w_dwt_afb2d_adjoint(const float* ll, long long ll_plane_stride, int ll_pitch, const float* highs,
                            float* y, long long y_plane_stride, int y_pitch,
                            int planes, int Hc, int Wc, int H, int W,
                            const float* fh_lo, const float* fh_hi, int Lh,
                            const float* fw_lo, const float* fw_hi, int Lw, int mode, void* stream);
int b200w_dwt_afb2d_adjoint_f64(const double* ll, long long ll_plane_stride, int ll_pitch, const double* highs,
                                double* y, long long y_plane_stride, int y_pitch,
                                int planes, int Hc, int Wc, int H, int W,
                                const double* fh_lo, const double* fh_hi, int Lh,
                                const double* fw_lo, const double* fw_hi, int Lw, int mode, void* stream);
int b200w_dwt_afb1d_adjoint(const float* lo, const float* hi, int rows, int K, float* y, int N,
                            const float* f0, const float* f1, int L, int mode, void* stream);
int b200w_dwt_afb1d_adjoint_f64(const double* lo, const double* hi, int rows, int K, double* y, int N,
                                const double* f0, const double* f1, int L, int mode, void* stream);

/* ---------------------------------------------------------------------------------------------
 * 3-D DWT levels (an addition beyond the reference; DWT3DForward / DWT3DInverse).  One filter pair acts along all
 * three axes.  Analysis = the 1-D analysis along W, then H, then D, each pass rounded to the element type; synthesis is
 * the reverse (along D, then the 2-D synthesis: H, then W).  Per axis the sizes follow b200w_dwt_coeff_len /
 * b200w_dwt_rec_len.  Band b = 4*aW + 2*aH + aD - 1 (aX = 1: high-pass along X), so bands 1, 3, 5 are the 2-D
 * lh, hl, hh of K1 low-passed along D and bands 0, 2, 4, 6 are high-pass along D.
 *   b200w_dwt_afb3d: x (volumes, D, H, W), volume stride x_vol_stride elements (>= D*H*W), last three dims dense
 *                    -> yl (volumes, Do, Ho, Wo) and highs (volumes, 7, Do, Ho, Wo), both contiguous.
 *                    f_lo, f_hi: stored (reversed) analysis taps, length L.
 *   b200w_dwt_sfb3d: yl (volumes, Dc, Hc, Wc) with volume stride yl_vol_stride (last three dims dense) and highs
 *                    (volumes, 7, Dc, Hc, Wc) contiguous, or NULL = zeros (then it is never read)
 *                    -> y (volumes, Do, Ho, Wo) contiguous.  Do / Ho / Wo may be smaller than the natural
 *                    b200w_dwt_rec_len sizes: the crop of the analysis backward pass.  g_lo, g_hi: synthesis taps.
 * Each also computes the other's backward pass when given the same stored filters.
 * A float32 level with L in {2, 4, 6, 8} is one fused kernel that reads its input once and writes every output once;
 * its workspace query returns 0.  Any other level takes the two-step route: the 2-D level (K1 / K2) over all
 * volumes*D planes plus a 1-D pass along D, with intermediates in `workspace` (caller-owned device memory of at least
 * the query's bytes; same arguments to both calls).  The _generic entries always take the two-step route (the A/B
 * reference of the parity tests); the _f64 entries take it in double.
 */
long long b200w_dwt_afb3d_workspace(const float* x, long long x_vol_stride, int volumes, int D, int H, int W, int L,
                                    int mode);
int b200w_dwt_afb3d(const float* x, long long x_vol_stride, float* yl, float* highs, int volumes, int D, int H, int W,
                    const float* f_lo, const float* f_hi, int L, int mode, void* workspace, long long workspace_bytes,
                    void* stream);
long long b200w_dwt_sfb3d_workspace(int volumes, int Dc, int Hc, int Wc, int Do, int Ho, int Wo, int L, int mode);
int b200w_dwt_sfb3d(const float* yl, long long yl_vol_stride, const float* highs, float* y, int volumes, int Dc,
                    int Hc, int Wc, int Do, int Ho, int Wo, const float* g_lo, const float* g_hi, int L, int mode,
                    void* workspace, long long workspace_bytes, void* stream);
long long b200w_dwt_afb3d_workspace_generic(const float* x, long long x_vol_stride, int volumes, int D, int H, int W,
                                            int L, int mode);
int b200w_dwt_afb3d_generic(const float* x, long long x_vol_stride, float* yl, float* highs, int volumes, int D, int H,
                            int W, const float* f_lo, const float* f_hi, int L, int mode, void* workspace,
                            long long workspace_bytes, void* stream);
long long b200w_dwt_sfb3d_workspace_generic(int volumes, int Dc, int Hc, int Wc, int Do, int Ho, int Wo, int L,
                                            int mode);
int b200w_dwt_sfb3d_generic(const float* yl, long long yl_vol_stride, const float* highs, float* y, int volumes,
                            int Dc, int Hc, int Wc, int Do, int Ho, int Wo, const float* g_lo, const float* g_hi, int L,
                            int mode, void* workspace, long long workspace_bytes, void* stream);
long long b200w_dwt_afb3d_workspace_f64(const double* x, long long x_vol_stride, int volumes, int D, int H, int W,
                                        int L, int mode);
int b200w_dwt_afb3d_f64(const double* x, long long x_vol_stride, double* yl, double* highs, int volumes, int D, int H,
                        int W, const double* f_lo, const double* f_hi, int L, int mode, void* workspace,
                        long long workspace_bytes, void* stream);
long long b200w_dwt_sfb3d_workspace_f64(int volumes, int Dc, int Hc, int Wc, int Do, int Ho, int Wo, int L, int mode);
int b200w_dwt_sfb3d_f64(const double* yl, long long yl_vol_stride, const double* highs, double* y, int volumes, int Dc,
                        int Hc, int Wc, int Do, int Ho, int Wo, const double* g_lo, const double* g_hi, int L,
                        int mode, void* workspace, long long workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * 1-D DTCWT levels (an addition beyond the reference; DTCWT1DForward / DTCWT1DInverse).  Signals are `rows`
 * independent rows; every output and the band-pass input are contiguous (rows, length) arrays.  Each call is one
 * kernel that computes both filters of the level (both trees at levels >= 2).  Taps are stored (reversed) host arrays.
 *   b200w_dtcwt1d_fwd_j1:     x (rows, n), row pitch x_pitch >= n -> lo, hi (rows, n); n even.
 *                             lo = colfilter(x, h0), hi = colfilter(x, h1) along the row, mode symmetric or zero.
 *                             h0 / h1 odd lengths L0 / L1.  hi may be NULL (skipped band-pass: nothing written).
 *   b200w_dtcwt1d_fwd_j2plus: x (rows, n), n % 4 == 0 -> lo, hi (rows, n / 2);
 *                             lo = coldfilt(x, h0b, h0a), hi = coldfilt(x, h1b, h1a, highpass); hi may be NULL.
 *   b200w_dtcwt1d_inv_j1:     lo (rows, n) with row pitch lo_pitch >= n, hi (rows, n) -> y (rows, n); n even.
 *                             y = colfilter(lo, g0) + colfilter(hi, g1).
 *   b200w_dtcwt1d_inv_j2plus: lo (rows, n / 2) with row pitch lo_pitch, hi (rows, n / 2) -> y (rows, n), n % 4 == 0;
 *                             y = colifilt(lo, g0b, g0a) + colifilt(hi, g1b, g1a, highpass).
 *   The inverses take NULL for lo and / or hi (zeros: that branch is skipped) and round each branch before the sum.
 * Errors: B200W_EARG for a NULL required pointer or a pitch below the row length, B200W_EMODE for a level-1 mode other
 * than zero / symmetric, B200W_ESIZE for n odd (j1) or n % 4 != 0 (j2plus), B200W_EFILTER for an even or longer than
 * B200W_MAX_TAPS level-1 filter or an odd / too long q-shift filter.  rows == 0 returns 0 without a launch.
 */
int b200w_dtcwt1d_fwd_j1(const float* x, long long x_pitch, int rows, int n, float* lo, float* hi,
                         const float* h0, int L0, const float* h1, int L1, int mode, void* stream);
int b200w_dtcwt1d_fwd_j2plus(const float* x, long long x_pitch, int rows, int n, float* lo, float* hi,
                             const float* h0a, const float* h1a, const float* h0b, const float* h1b, int m,
                             void* stream);
int b200w_dtcwt1d_inv_j1(const float* lo, long long lo_pitch, const float* hi, int rows, int n, float* y,
                         const float* g0, int L0, const float* g1, int L1, int mode, void* stream);
int b200w_dtcwt1d_inv_j2plus(const float* lo, long long lo_pitch, const float* hi, int rows, int n, float* y,
                             const float* g0a, const float* g1a, const float* g0b, const float* g1b, int m,
                             void* stream);
int b200w_dtcwt1d_fwd_j1_f64(const double* x, long long x_pitch, int rows, int n, double* lo, double* hi,
                             const double* h0, int L0, const double* h1, int L1, int mode, void* stream);
int b200w_dtcwt1d_fwd_j2plus_f64(const double* x, long long x_pitch, int rows, int n, double* lo, double* hi,
                                 const double* h0a, const double* h1a, const double* h0b, const double* h1b, int m,
                                 void* stream);
int b200w_dtcwt1d_inv_j1_f64(const double* lo, long long lo_pitch, const double* hi, int rows, int n, double* y,
                             const double* g0, int L0, const double* g1, int L1, int mode, void* stream);
int b200w_dtcwt1d_inv_j2plus_f64(const double* lo, long long lo_pitch, const double* hi, int rows, int n, double* y,
                                 const double* g0a, const double* g1a, const double* g0b, const double* g1b, int m,
                                 void* stream);

/* ---------------------------------------------------------------------------------------------
 * 1-D scattering levels (ScatLayer1D / ScatLayer1Dj2): a 1-D DTCWT forward level with the scattering epilogue, one
 * kernel.  x is N * C rows of length n with row pitch x_pitch >= n.  Element (b, c, i) of an output of row length m is
 * at base + b * bstride + c * m + i, with bstride >= C * m, so an output can be one slot s of a (N, S, C, m) tensor
 * (base + s * C * m, bstride S * C * m).  With (re, im) = (hi[2q], hi[2q + 1]) the band-pass pairs of the level and
 * b = (T)magbias, b2 = (T)(magbias * magbias) (product in double), every operation rounded:
 *   mag[q] = sqrt((re * re + im * im) + b2) - b;  dre[q] = re / r, dim[q] = im / r, r the rounded root;
 *   pool(lo)[q] = (lo[2q] + lo[2q + 1]) * 0.5.
 *   b200w_scat1d_j1:     lo, hi = colfilter(x, h0), colfilter(x, h1), mode symmetric or zero; n even.  Writes
 *                        pool(lo) (m = n / 2) when pool_lo, else lo itself (m = n); mag (m = n / 2).
 *   b200w_scat1d_j2plus: lo, hi = coldfilt(x, h0b, h0a), coldfilt(x, h1b, h1a, highpass); n % 4 == 0.  Writes pool(lo)
 *                        and mag (m = n / 4).
 *   dre and dim (row length of mag) are both NULL (not written) or both given.
 * Errors as b200w_dtcwt1d_*: B200W_EARG for a NULL required pointer, only one of dre / dim, a pitch or batch stride
 * below its row block; B200W_EMODE for a level-1 mode other than zero / symmetric; B200W_ESIZE for negative N or C,
 * N * C above INT_MAX, n odd (j1) or n % 4 != 0 (j2plus); B200W_EFILTER for a bad filter length.  N * C == 0 returns 0
 * without a launch.
 */
int b200w_scat1d_j1(const float* x, long long x_pitch, int N, int C, int n, float* lo, long long lo_bstride, int pool_lo,
                    float* mag, long long mag_bstride, float* dre, long long dre_bstride, float* dim,
                    long long dim_bstride, const float* h0, int L0, const float* h1, int L1, int mode, double magbias,
                    void* stream);
int b200w_scat1d_j2plus(const float* x, long long x_pitch, int N, int C, int n, float* lo, long long lo_bstride,
                        float* mag, long long mag_bstride, float* dre, long long dre_bstride, float* dim,
                        long long dim_bstride, const float* h0a, const float* h1a, const float* h0b, const float* h1b,
                        int m, double magbias, void* stream);
int b200w_scat1d_j1_f64(const double* x, long long x_pitch, int N, int C, int n, double* lo, long long lo_bstride,
                        int pool_lo, double* mag, long long mag_bstride, double* dre, long long dre_bstride,
                        double* dim, long long dim_bstride, const double* h0, int L0, const double* h1, int L1,
                        int mode, double magbias, void* stream);
int b200w_scat1d_j2plus_f64(const double* x, long long x_pitch, int N, int C, int n, double* lo, long long lo_bstride,
                            double* mag, long long mag_bstride, double* dre, long long dre_bstride, double* dim,
                            long long dim_bstride, const double* h0a, const double* h1a, const double* h0b,
                            const double* h1b, int m, double magbias, void* stream);

/* ---------------------------------------------------------------------------------------------
 * 2-D wavelet packet levels (csrc/wpt2d.cu).  One DWT analysis / synthesis level (the arithmetic of
 * b200w_dwt_afb2d / b200w_dwt_sfb2d) applied to every plane, in the packet layout: the four children
 * of plane p (ll, lh, hl, hh) are nodes 4p .. 4p+3, so one level's output is the next level's input.
 *   b200w_wpt_afb2d: x planes (plane stride, row pitch) -> node 4p + b at y + (4p + b) * y_node_stride,
 *                    rows y_pitch apart; Ho, Wo = b200w_dwt_coeff_len of H, W.
 *   b200w_wpt_sfb2d: c contiguous (planes * 4, Hc, Wc) -> y planes (plane stride, row pitch) of Ho x Wo,
 *                    Ho / Wo at most b200w_dwt_rec_len of Hc / Wc (smaller values crop, as in the
 *                    analysis backward pass).
 * The route is chosen per call from the plane size, filter lengths and alignment: a packed small-plane
 * kernel, the streaming kernel (float32, Lw == Lh <= 20) or the generic tile kernel (every case; the
 * only one the _generic entries run).  Errors: B200W_EMODE for an unknown mode; B200W_EARG for a NULL
 * pointer, a pitch below its row length, or a node / plane stride below Ho * pitch; B200W_ESIZE for bad
 * sizes or a grid that is too large; B200W_EFILTER for a length outside 2 .. B200W_MAX_TAPS (Lw != Lh is
 * allowed).  planes == 0 returns 0 without a launch.
 */
int b200w_wpt_afb2d(const float* x, long long x_plane_stride, int x_pitch, float* y, long long y_node_stride,
                    int y_pitch, int planes, int H, int W, const float* fw_lo, const float* fw_hi, int Lw,
                    const float* fh_lo, const float* fh_hi, int Lh, int mode, void* stream);
int b200w_wpt_afb2d_generic(const float* x, long long x_plane_stride, int x_pitch, float* y, long long y_node_stride,
                            int y_pitch, int planes, int H, int W, const float* fw_lo, const float* fw_hi, int Lw,
                            const float* fh_lo, const float* fh_hi, int Lh, int mode, void* stream);
int b200w_wpt_afb2d_f64(const double* x, long long x_plane_stride, int x_pitch, double* y, long long y_node_stride,
                        int y_pitch, int planes, int H, int W, const double* fw_lo, const double* fw_hi, int Lw,
                        const double* fh_lo, const double* fh_hi, int Lh, int mode, void* stream);
int b200w_wpt_sfb2d(const float* c, float* y, long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc,
                    int Ho, int Wo, const float* gh_lo, const float* gh_hi, int Lh, const float* gw_lo,
                    const float* gw_hi, int Lw, int mode, void* stream);
int b200w_wpt_sfb2d_generic(const float* c, float* y, long long y_plane_stride, int y_pitch, int planes, int Hc,
                            int Wc, int Ho, int Wo, const float* gh_lo, const float* gh_hi, int Lh, const float* gw_lo,
                            const float* gw_hi, int Lw, int mode, void* stream);
int b200w_wpt_sfb2d_f64(const double* c, double* y, long long y_plane_stride, int y_pitch, int planes, int Hc, int Wc,
                        int Ho, int Wo, const double* gh_lo, const double* gh_hi, int Lh, const double* gw_lo,
                        const double* gw_hi, int Lw, int mode, void* stream);

/* ---------------------------------------------------------------------------------------------
 * DTCWT.  "highs" is the reference's 6-D complex band-pass tensor; because o_dim / ri_dim are
 * configurable (dtcwt/transform_funcs.py:10-58) it is described by six ELEMENT strides
 * hs[6] = {n, c, orientation, row, col, real/imag}.  Default layout (N,C,6,H/2,W/2,2) is the
 * fast path.  Orientation order 15,45,75,105,135,165 degrees (transform_funcs.py:61-72).
 *
 * K3  level-1 forward.                     Replaces FWD_J1.forward, dtcwt/transform_funcs.py:346-358
 *     (fwd_j1 :98-121 = rowfilter x2, colfilter x4 (dtcwt/lowlevel.py:70-94), q2c :243-260).
 *   x   (N*C, H, W) pitched, H and W even;  ll (N*C, H, W) pitched
 *   highs: band-pass output at (H/2, W/2) or NULL when skip_hps.
 *   h0,h1: stored (reversed) level-1 filters, odd lengths L0, L1.
 *   mode: B200W_MODE_SYMMETRIC -> symmetric extension, anything else -> zero padding
 *         (dtcwt/lowlevel.py:75-79).
 * Also INV_J1.backward (:434-449) when given g0o/g1o.
 */
int b200w_dtcwt_fwd_j1(const float* x, long long x_plane_stride, int x_pitch,
                       float* ll, long long ll_plane_stride, int ll_pitch,
                       float* highs, const long long hs[6],
                       int N, int C, int H, int W,
                       const float* h0, int L0, const float* h1, int L1,
                       int mode, void* stream);

/* K4  level>=2 forward.                    Replaces FWD_J2PLUS.forward, transform_funcs.py:380-392
 *     (fwd_j2plus :226-249 = rowdfilt x2, coldfilt x4 (dtcwt/lowlevel.py:97-151), q2c).
 *   x (N*C,H,W) with H%4==0 and W%4==0 (else B200W_ESIZE, reference ValueError lowlevel.py:102-104);
 *   ll (N*C,H/2,W/2); highs at (H/4,W/4) or NULL when skip_hps.
 *   h0a,h1a,h0b,h1b: stored (reversed) q-shift filters, common even length m.
 *   Always symmetric extension (transform_funcs.py:381).
 * Also INV_J2PLUS.backward (:471-488) with a<->b swapped by the caller.
 */
int b200w_dtcwt_fwd_j2plus(const float* x, long long x_plane_stride, int x_pitch,
                           float* ll, long long ll_plane_stride, int ll_pitch,
                           float* highs, const long long hs[6],
                           int N, int C, int H, int W,
                           const float* h0a, const float* h1a,
                           const float* h0b, const float* h1b, int m,
                           void* stream);

/* K3+K4  levels 1 and 2 forward in one call: what b200w_dtcwt_fwd_j1 followed by b200w_dtcwt_fwd_j2plus on its
 *     low-pass computes (bit for bit), without returning the level-1 low-pass.
 *   x (N*C,H,W) pitched with H%4==0 and W%4==0 (else B200W_ESIZE); ll2 (N*C,H/2,W/2) pitched;
 *   highs0 at (H/2,W/2) or NULL; highs1 at (H/4,W/4) or NULL; hs0 / hs1 their element strides as above.
 *   h0o,h1o: stored level-1 filters (odd lengths L0, L1); h0a,h1a,h0b,h1b: stored q-shift filters (length m);
 *   mode: level 1's extension as for b200w_dtcwt_fwd_j1.
 *   When the fused kernel covers the call (highs0 given, 16-byte aligned rows, a compiled filter pair, a plane width
 *   the kernel fits) the level-1 low-pass stays on chip and b200w_dtcwt_fwd_j12_workspace returns 0; otherwise it
 *   returns the bytes of a float32 (N*C,H,W) low-pass and the two level kernels run through the caller's workspace
 *   (B200W_EARG when it is missing or smaller).  The _generic form always runs the two generic tile levels and
 *   always needs that workspace.  Validation as b200w_dtcwt_fwd_j1 / b200w_dtcwt_fwd_j2plus; N*C == 0 is a no-op.
 */
long long b200w_dtcwt_fwd_j12_workspace(const float* x, long long x_plane_stride, int x_pitch, const float* highs0,
                                        int N, int C, int H, int W, int L0, int L1, int m);
int b200w_dtcwt_fwd_j12(const float* x, long long x_plane_stride, int x_pitch,
                        float* ll2, long long ll2_plane_stride, int ll2_pitch,
                        float* highs0, const long long hs0[6], float* highs1, const long long hs1[6],
                        int N, int C, int H, int W,
                        const float* h0o, int L0, const float* h1o, int L1,
                        const float* h0a, const float* h1a, const float* h0b, const float* h1b, int m,
                        int mode, void* workspace, long long workspace_bytes, void* stream);

/* K5  level-1 inverse.                     Replaces INV_J1.forward, transform_funcs.py:419-431
 *     (inv_j1 :152-184 = c2q (dtcwt/lowlevel.py:263-295), colfilter x4, rowfilter x2).
 *   ll (N*C,H,W) pitched or NULL (treated as zeros); highs at (H/2,W/2) or NULL (low-pass only
 *   path, which the reference runs with symmetric extension regardless of mode, :159);
 *   y (N*C,H,W).  g0,g1 stored level-1 synthesis filters (odd lengths).
 * Also FWD_J1.backward (:361-374) when given h0o/h1o.
 */
int b200w_dtcwt_inv_j1(const float* ll, long long ll_plane_stride, int ll_pitch,
                       const float* highs, const long long hs[6],
                       float* y, long long y_plane_stride, int y_pitch,
                       int N, int C, int H, int W,
                       const float* g0, int L0, const float* g1, int L1,
                       int mode, void* stream);

/* K6  level>=2 inverse.                    Replaces INV_J2PLUS.forward, transform_funcs.py:455-468
 *     (inv_j2plus :279-307 = c2q, colifilt x4, rowifilt x2 (dtcwt/lowlevel.py:154-239)).
 *   ll (N*C,H,W) or NULL; highs at (H/2,W/2) or NULL; y (N*C,2H,2W).  H, W even.
 *   g0a,g1a,g0b,g1b stored q-shift synthesis filters, common even length m.
 * Also FWD_J2PLUS.backward (:395-413) with a<->b swapped by the caller.
 */
int b200w_dtcwt_inv_j2plus(const float* ll, long long ll_plane_stride, int ll_pitch,
                           const float* highs, const long long hs[6],
                           float* y, long long y_plane_stride, int y_pitch,
                           int N, int C, int H, int W,
                           const float* g0a, const float* g1a,
                           const float* g0b, const float* g1b, int m,
                           void* stream);

/* K7  ScatLayer forward.                   Replaces ScatLayerj1_f.forward (combine_colour=False),
 *     scatternet/lowlevel.py:76-111: level-1 DTCWT (o_dim=1) -> 2x2 mean of ll ->
 *     sqrt(re^2+im^2+b^2)-b -> stacked (N,7,C,H/2,W/2).
 *   x (N,C,H,W) contiguous, H and W even; z (N,7,C,H/2,W/2) contiguous.
 *   dre_dr / dim_dr: optional (N,6,C,H/2,W/2) outputs re/r and im/r saved for the backward
 *   pass (:96-99); pass NULL when no gradient is needed.
 */
int b200w_scat_j1(const float* x, float* z, float* dre_dr, float* dim_dr,
                  int N, int C, int H, int W,
                  const float* h0, int L0, const float* h1, int L1,
                  int mode, float magbias, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Multi-GPU.  Every (n, c) plane is transformed independently (depthwise filters, no halo between planes:
 * reference dwt/lowlevel.py:143,164,168; dtcwt/lowlevel.py:77,111), so the batch shards over the GPUs of a
 * box with NO exchange during compute; the one collective of the path is the all-gather of the returned
 * tensors along dim 0 after the last level.  One process per GPU; the communicator is an explicit handle
 * (no hidden global state).  NCCL is bound at run time; without it these return B200W_ENOTIMPL.
 *   b200w_comm_unique_id  rank 0 creates the 128-byte NCCL id and hands it to the other ranks out of band
 *                         (the Python shell broadcasts it through torch.distributed)
 *   b200w_comm_init       collective over all ranks; binds the communicator to the CURRENT CUDA device
 *   b200w_allgather       recv[r*count .. (r+1)*count) = rank r's send[0 .. count)  (fp32 elements), asynchronous
 *                         on `stream` (pass the compute stream: the gather then simply follows the last level)
 */
typedef struct b200w_comm b200w_comm;
int b200w_comm_unique_id(void* id128);
int b200w_comm_init(b200w_comm** comm, int rank, int world, const void* id128);
int b200w_comm_destroy(b200w_comm* comm);
int b200w_allgather(b200w_comm* comm, const float* send, float* recv, long long count, void* stream);
const char* b200w_comm_last_error(void);

/* ---------------------------------------------------------------------------------------------
 * Generic-kernel variants.  Every entry point above picks a specialised streaming kernel when one
 * exists for the filter lengths / layout / alignment it is given and otherwise runs the generic tile
 * kernel (any filter length <= B200W_MAX_TAPS, any mode, any layout).  The *_generic symbols take the
 * same arguments and always run the generic tile kernel: an independent second implementation of the
 * same arithmetic, used by the parity tests for A/B checks (selection is per call -- the library keeps
 * no mode switch or any other global mutable state).
 */
int b200w_dwt_afb2d_generic(const float* x, long long x_plane_stride, int x_pitch,
                            float* ll, long long ll_plane_stride, int ll_pitch, float* highs,
                            int planes, int H, int W,
                            const float* fw_lo, const float* fw_hi, int Lw,
                            const float* fh_lo, const float* fh_hi, int Lh, int mode, void* stream);
int b200w_dwt_forward_generic(const float* x, long long x_plane_stride, int x_pitch,
                              int planes, int H, int W, int J, float* yl, float* const* highs,
                              const float* fw_lo, const float* fw_hi, int Lw,
                              const float* fh_lo, const float* fh_hi, int Lh,
                              int mode, void* workspace, long long workspace_bytes, void* stream);
int b200w_dwt_sfb2d_generic(const float* ll, long long ll_plane_stride, int ll_pitch, const float* highs,
                            float* y, long long y_plane_stride, int y_pitch,
                            int planes, int Hc, int Wc, int Ho, int Wo,
                            const float* gh_lo, const float* gh_hi, int Lh,
                            const float* gw_lo, const float* gw_hi, int Lw, int mode, void* stream);
int b200w_dtcwt_fwd_j1_generic(const float* x, long long x_plane_stride, int x_pitch,
                               float* ll, long long ll_plane_stride, int ll_pitch,
                               float* highs, const long long hs[6], int N, int C, int H, int W,
                               const float* h0, int L0, const float* h1, int L1, int mode, void* stream);
int b200w_dtcwt_fwd_j2plus_generic(const float* x, long long x_plane_stride, int x_pitch,
                                   float* ll, long long ll_plane_stride, int ll_pitch,
                                   float* highs, const long long hs[6], int N, int C, int H, int W,
                                   const float* h0a, const float* h1a, const float* h0b, const float* h1b,
                                   int m, void* stream);
int b200w_dtcwt_fwd_j12_generic(const float* x, long long x_plane_stride, int x_pitch,
                                float* ll2, long long ll2_plane_stride, int ll2_pitch,
                                float* highs0, const long long hs0[6], float* highs1, const long long hs1[6],
                                int N, int C, int H, int W,
                                const float* h0o, int L0, const float* h1o, int L1,
                                const float* h0a, const float* h1a, const float* h0b, const float* h1b, int m,
                                int mode, void* workspace, long long workspace_bytes, void* stream);
int b200w_dtcwt_inv_j1_generic(const float* ll, long long ll_plane_stride, int ll_pitch,
                               const float* highs, const long long hs[6],
                               float* y, long long y_plane_stride, int y_pitch, int N, int C, int H, int W,
                               const float* g0, int L0, const float* g1, int L1, int mode, void* stream);
int b200w_dtcwt_inv_j2plus_generic(const float* ll, long long ll_plane_stride, int ll_pitch,
                                   const float* highs, const long long hs[6],
                                   float* y, long long y_plane_stride, int y_pitch, int N, int C, int H, int W,
                                   const float* g0a, const float* g1a, const float* g0b, const float* g1b,
                                   int m, void* stream);
int b200w_scat_j1_generic(const float* x, float* z, float* dre_dr, float* dim_dr, int N, int C, int H, int W,
                          const float* h0, int L0, const float* h1, int L1, int mode, float magbias, void* stream);

/* ---------------------------------------------------------------------------------------------
 * float64 variants.  The reference computes in torch's default dtype (dwt/lowlevel.py:972,
 * dtcwt/lowlevel.py:67), so double-precision modules work there.  Here double precision runs the
 * generic tile kernels (and the 1-D row kernels) compiled for `double`: same arguments as the
 * float32 entry points with `double` in place of `float`, same return codes, same stream semantics.
 * (The streaming / pyramid fast paths and b200w_dwt_forward are float32-only.)
 */
int b200w_dwt_afb2d_f64(const double* x, long long x_plane_stride, int x_pitch,
                        double* ll, long long ll_plane_stride, int ll_pitch, double* highs,
                        int planes, int H, int W,
                        const double* fw_lo, const double* fw_hi, int Lw,
                        const double* fh_lo, const double* fh_hi, int Lh, int mode, void* stream);
int b200w_dwt_sfb2d_f64(const double* ll, long long ll_plane_stride, int ll_pitch, const double* highs,
                        double* y, long long y_plane_stride, int y_pitch,
                        int planes, int Hc, int Wc, int Ho, int Wo,
                        const double* gh_lo, const double* gh_hi, int Lh,
                        const double* gw_lo, const double* gw_hi, int Lw, int mode, void* stream);
int b200w_dwt_afb1d_f64(const double* x, long long x_pitch, int rows, int N, double* lo, double* hi,
                        const double* f0, const double* f1, int L, int mode, void* stream);
int b200w_dwt_sfb1d_f64(const double* lo, const double* hi, int rows, int K, double* y, int Nout,
                        const double* g0, const double* g1, int L, int mode, void* stream);
int b200w_dtcwt_fwd_j1_f64(const double* x, long long x_plane_stride, int x_pitch,
                           double* ll, long long ll_plane_stride, int ll_pitch,
                           double* highs, const long long hs[6], int N, int C, int H, int W,
                           const double* h0, int L0, const double* h1, int L1, int mode, void* stream);
int b200w_dtcwt_fwd_j2plus_f64(const double* x, long long x_plane_stride, int x_pitch,
                               double* ll, long long ll_plane_stride, int ll_pitch,
                               double* highs, const long long hs[6], int N, int C, int H, int W,
                               const double* h0a, const double* h1a, const double* h0b, const double* h1b,
                               int m, void* stream);
int b200w_dtcwt_inv_j1_f64(const double* ll, long long ll_plane_stride, int ll_pitch,
                           const double* highs, const long long hs[6],
                           double* y, long long y_plane_stride, int y_pitch, int N, int C, int H, int W,
                           const double* g0, int L0, const double* g1, int L1, int mode, void* stream);
int b200w_dtcwt_inv_j2plus_f64(const double* ll, long long ll_plane_stride, int ll_pitch,
                               const double* highs, const long long hs[6],
                               double* y, long long y_plane_stride, int y_pitch, int N, int C, int H, int W,
                               const double* g0a, const double* g1a, const double* g0b, const double* g1b,
                               int m, void* stream);
int b200w_scat_j1_f64(const double* x, double* z, double* dre_dr, double* dim_dr, int N, int C, int H, int W,
                      const double* h0, int L0, const double* h1, int L1, int mode, double magbias, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Standalone 1-D DTCWT primitives (the reference's low-level API; in the transforms these passes are
 * fused inside the per-level kernels).  x: (planes, H, W) contiguous; y: contiguous output.
 *   b200w_dtcwt_filter  = colfilter (along_w = 0) / rowfilter (along_w = 1), reference
 *                         dtcwt/lowlevel.py:70-94: y[n] = sum_j h[j] x[ext(n + j - L/2)], ext = symmetric
 *                         or zero padding; ANY length L -- an even L yields N + 1 outputs along the
 *                         filtered dimension (the reference's behaviour, tests/test_colfilter.py:52-61).
 *   b200w_dtcwt_dfilt   = coldfilt / rowdfilt (:97-151): (ha, hb) even length m, filtered size % 4 == 0,
 *                         output half size.
 *   b200w_dtcwt_ifilt   = colifilt / rowifilt (:154-239): filtered size % 2 == 0, output double size.
 * Taps are host pointers in stored (reversed) order, as everywhere in this ABI.
 */
int b200w_dtcwt_filter(const float* x, float* y, int planes, int H, int W, const float* h, int L,
                       int symmetric, int along_w, void* stream);
int b200w_dtcwt_dfilt(const float* x, float* y, int planes, int H, int W, const float* ha, const float* hb,
                      int m, int highpass, int along_w, void* stream);
int b200w_dtcwt_ifilt(const float* x, float* y, int planes, int H, int W, const float* ha, const float* hb,
                      int m, int highpass, int along_w, void* stream);
int b200w_dtcwt_filter_f64(const double* x, double* y, int planes, int H, int W, const double* h, int L,
                           int symmetric, int along_w, void* stream);
int b200w_dtcwt_dfilt_f64(const double* x, double* y, int planes, int H, int W, const double* ha,
                          const double* hb, int m, int highpass, int along_w, void* stream);
int b200w_dtcwt_ifilt_f64(const double* x, double* y, int planes, int H, int W, const double* ha,
                          const double* hb, int m, int highpass, int along_w, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200WAVE_H */
