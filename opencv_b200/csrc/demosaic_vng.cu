// demosaic_vng.cu -- cv::cvtColor / cv::demosaicing with Variable Number of Gradients, codes COLOR_BayerBG/GB/RG/GR2BGR_VNG = 62..65
// (the 2RGB_VNG names are the same numbers permuted), 8-bit mosaic, 3-channel destination.
//
// Reference: Bayer2RGB_VNG_8u (demosaicing.cpp:1059-1587).  Per mosaic row it computes seven u16 gradient planes of the 3 x 3
// neighbourhood (:1090-1154); per pixel of rows 2 .. H-5 and columns 2 .. W-3 it sums them into eight directional gradients, takes the
// directions below T = minGrad + max(maxGrad / 2, 1) (ng >= 1 of them) and adds the mean colour differences over those directions,
// scaled and rounded half to even, to the sample (:1172-1330).  The rest is copied: columns 0-1 / W-2, W-1 from columns 2 / W-3, then
// rows 0-1 / H-4 .. H-1 from rows 2 / H-5 (:1569-1586), so the pixel at (y, x) is the value computed for (clamp(y, 2, H-5), clamp(x, 2, W-3)).
// The reference advances its mosaic pointer by two rows before that loop (:1083) and then indexes it with the destination row, so
// destination row y is computed from the mosaic around row y + 2 (with row y's pattern, the same parity): the kernel does the same.
// All integer up to the scaling, whose factor depends on the reference's arm (vng_scale below): its 8-pixel vector body and its scalar
// head / tail differ at ng == 7.  vng_planes / vng_pixel / vng_simd_arm use nothing a host build lacks, so that the CPU suite runs them
// (tests/test_bayer_reference.py).  Images with min(W, H) < 8 take the reference's bilinear Bayer2RGB_, which reads the VNG code as
// COLOR_BayerRG2BGR whatever the pattern (:1071-1075, :1026-1029): demosaic_bilinear with code 48.
//
// Kernel: one block per 64 x 32 pixels; the mosaic tile with a 2-pixel apron is staged in shared memory, the seven planes are computed
// once for the tile with a 1-pixel apron (u16, shared), and each thread evaluates 8 consecutive pixels of one row, stored as one
// 24-byte write when aligned.
#include "common.cuh"
#include "bytes.cuh"

namespace b200cv {

// the factor that turns a sum of ng colour differences into a mean difference (1 / (2 ng)).  The scalar loop multiplies by the table
// scale[] = {0, 0.5f, 0.25f, 0.1666666666667f, 0.125f, 0.1f, 0.08333333333f, 0.0714286f, 0.0625f} (:1159), the vector body by
// 0.5f / (float)ng (:1530).  As float32 the two agree for every ng except 7 (0.0714286f vs 0.071428575f).
__device__ __forceinline__ float vng_scale(int ng, bool simd)
{
    return ng == 1 ? 0.5f : ng == 2 ? 0.25f : ng == 3 ? 0.1666666666667f : ng == 4 ? 0.125f : ng == 5 ? 0.1f : ng == 6 ? 0.08333333333f
         : ng == 7 ? (simd ? 0.071428575f : 0.0714286f) : 0.0625f;
}

// does the reference's 8-pixel vector body compute column x of a row whose column 2 is a green site (green_at_2) or not?  The scalar
// head runs columns 2 .. limit-1 with limit = 3 for a green column 2 and 2 otherwise (:1165), so the body starts on a red / blue site;
// it runs while its first column is <= W - 10 (:1342); the scalar tail finishes the row.
__device__ __forceinline__ bool vng_simd_arm(int x, bool green_at_2, int W)
{
    const int s = green_at_2 ? 3 : 2;
    if (W - 10 < s) return false;
    return x >= s && x < s + ((W - 10 - s) / 8 + 1) * 8;
}

// the seven gradient planes at one mosaic site q (row pitch ms), written to p[0], p[pk], .. p[6 * pk] (:1138-1153); every value is <= 1020
__device__ __forceinline__ void vng_planes(const uchar* q, int ms, unsigned short* p, int pk)
{
    const int s1 = q[-ms - 1], s2 = q[-ms], s3 = q[-ms + 1], s4 = q[-1], s6 = q[1], s7 = q[ms - 1], s8 = q[ms], s9 = q[ms + 1];
    const int b2 = abs(s3 - s7) * 2, b3 = abs(s1 - s9) * 2;
    p[0] = (unsigned short)(abs(s1 - s7) + abs(s2 - s8) * 2 + abs(s3 - s9));
    p[pk] = (unsigned short)(abs(s1 - s3) + abs(s4 - s6) * 2 + abs(s7 - s9));
    p[2 * pk] = (unsigned short)b2;
    p[3 * pk] = (unsigned short)b3;
    p[4 * pk] = (unsigned short)(b2 + abs(s2 - s4) + abs(s8 - s6));
    p[5 * pk] = (unsigned short)(b3 + abs(s2 - s6) + abs(s8 - s4));
    p[6 * pk] = (unsigned short)((s2 + s4 + s6 + s8) >> 1);
}

// One output pixel at a computed site.  m: the mosaic at the site (row pitch ms bytes); p: plane 0 at the site (row pitch pr, plane
// stride pk elements; planes 0..6 = vertical, horizontal, the two diagonals x 2, the diagonals plus edge terms, half the 4-neighbour
// sum).  Returns the reference's R, G, B (:1250-1252, :1322-1324): c is the colour of the row's red / blue sites (the sample there, the
// horizontal neighbours' colour at a green site), g green, o the other colour.  The caller writes o to channel blueIdx, c to blueIdx ^ 2.
__device__ __forceinline__ void vng_pixel(const uchar* m, int ms, const unsigned short* p, int pr, int pk, bool green, bool simd,
                                                   int& c, int& g, int& o)
{
    const unsigned short *P0 = p, *P1 = p + pk, *P2 = p + 2 * pk, *P3 = p + 3 * pk, *P4 = p + 4 * pk, *P5 = p + 5 * pk, *P6 = p + 6 * pk;
#define S(dy, dx) ((int)m[(dy) * ms + (dx)])
    const int gN = P0[-pr] + P0[0], gS = P0[0] + P0[pr], gW = P1[-1] + P1[0], gE = P1[0] + P1[1];
    int gNE, gSW, gNW, gSE;
    if (green) {
        gNE = P2[-pr] + P2[-pr + 1] + P2[0] + P2[1];
        gSW = P2[0] + P2[-1] + P2[pr] + P2[pr - 1];
        gNW = P3[-pr] + P3[-pr - 1] + P3[0] + P3[-1];
        gSE = P3[0] + P3[1] + P3[pr] + P3[pr + 1];
    } else {
        gNE = P4[-pr + 1] + P4[0];
        gSW = P4[0] + P4[pr - 1];
        gNW = P5[-pr - 1] + P5[0];
        gSE = P5[0] + P5[pr + 1];
    }
    const int mn = min(min(min(gN, gS), min(gW, gE)), min(min(gNE, gSW), min(gNW, gSE)));
    const int mx = max(max(max(gN, gS), max(gW, gE)), max(max(gNE, gSW), max(gNW, gSE)));
    const int T = mn + max(mx >> 1, 1);
    const int c0 = S(0, 0);
    int a = 0, b = 0, d = 0, ng = 0;        // red / blue site: (Rs, Gs, Bs); green site: (Gs, Rs, Bs) -- a always holds the sample's colour
    if (!green) {
        if (gN < T) { a += S(-2, 0) + c0; b += S(-1, 0) * 2; d += S(-1, -1) + S(-1, 1); ng++; }
        if (gS < T) { a += S(2, 0) + c0; b += S(1, 0) * 2; d += S(1, -1) + S(1, 1); ng++; }
        if (gW < T) { a += S(0, -2) + c0; b += S(0, -1) * 2; d += S(-1, -1) + S(1, -1); ng++; }
        if (gE < T) { a += S(0, 2) + c0; b += S(0, 1) * 2; d += S(-1, 1) + S(1, 1); ng++; }
        if (gNE < T) { a += S(-2, 2) + c0; b += P6[-pr + 1]; d += S(-1, 1) * 2; ng++; }
        if (gSW < T) { a += S(2, -2) + c0; b += P6[pr - 1]; d += S(1, -1) * 2; ng++; }
        if (gNW < T) { a += S(-2, -2) + c0; b += P6[-pr - 1]; d += S(-1, -1) * 2; ng++; }
        if (gSE < T) { a += S(2, 2) + c0; b += P6[pr + 1]; d += S(1, 1) * 2; ng++; }
    } else {
        if (gN < T) { b += S(-2, -1) + S(-2, 1); a += S(-2, 0) + c0; d += S(-1, 0) * 2; ng++; }
        if (gS < T) { b += S(2, -1) + S(2, 1); a += S(2, 0) + c0; d += S(1, 0) * 2; ng++; }
        if (gW < T) { b += S(0, -1) * 2; a += S(0, -2) + c0; d += S(-1, -2) + S(1, -2); ng++; }
        if (gE < T) { b += S(0, 1) * 2; a += S(0, 2) + c0; d += S(-1, 2) + S(1, 2); ng++; }
        if (gNE < T) { b += S(-2, 1) + S(0, 1); a += S(-1, 1) * 2; d += S(-1, 0) + S(-1, 2); ng++; }
        if (gSW < T) { b += S(2, -1) + S(0, -1); a += S(1, -1) * 2; d += S(1, 0) + S(1, -2); ng++; }
        if (gNW < T) { b += S(-2, -1) + S(0, -1); a += S(-1, -1) * 2; d += S(-1, -2) + S(-1, 0); ng++; }
        if (gSE < T) { b += S(2, 1) + S(0, 1); a += S(1, 1) * 2; d += S(1, 2) + S(1, 0); ng++; }
    }
#undef S
    // every sum is <= 8 * 510, so (float)(b - a) is exact; one float32 product, rounded half to even (cvRound / v_round)
    const float f = vng_scale(ng, simd);
    const int db = c0 + __float2int_rn(__fmul_rn((float)(b - a), f));
    const int dd = c0 + __float2int_rn(__fmul_rn((float)(d - a), f));
    c = min(max(green ? db : c0, 0), 255);
    g = min(max(green ? c0 : db, 0), 255);
    o = min(max(dd, 0), 255);
}

#ifndef B200CV_HOST_EMULATION
namespace {

constexpr int VNG_TW = 64, VNG_TH = 32;                       // computed pixels per block
constexpr int VNG_MW = VNG_TW + 4, VNG_MH = VNG_TH + 4;       // mosaic tile, 2-pixel apron
constexpr int VNG_PW = VNG_TW + 2, VNG_PH = VNG_TH + 2;       // plane tile, 1-pixel apron
constexpr int VNG_PK = VNG_PW * VNG_PH;

// blue0: destination channel of the blue colour in row 2 (0 or 2); green0: column 2 of row 2 is a green site
__global__ void __launch_bounds__(256) bayer_vng_kernel(Img src, Img dst, int W, int H, int blue0, int green0)
{
    __shared__ uchar sm[VNG_MH * VNG_MW];
    __shared__ unsigned short sp[7 * VNG_PK];
    const int f = blockIdx.z, tid = threadIdx.x;
    const int x0 = blockIdx.x * VNG_TW, y0 = blockIdx.y * VNG_TH;
    // computed pixels of this block: rows by .. by + VNG_TH - 1 at most, columns bx .. bx + VNG_TW - 1 (clamp is monotone and 1-Lipschitz);
    // their mosaic sites are rows by + 2 .., so the staged tile starts at mosaic row by and column bx - 2
    const int bx = min(max(x0, 2), W - 3), by = min(max(y0, 2), H - 5);
    for (int k = tid; k < VNG_MH * VNG_MW; k += 256) {
        const int r = k / VNG_MW, cc = k - r * VNG_MW;
        sm[k] = src.row<uchar>(f, min(by + r, H - 1))[min(bx - 2 + cc, W - 1)];         // rows shifted by 2 (see above); clamped entries are never used
    }
    __syncthreads();
    for (int k = tid; k < VNG_PK; k += 256) {
        const int r = k / VNG_PW, cc = k - r * VNG_PW;
        vng_planes(sm + (r + 1) * VNG_MW + cc + 1, VNG_MW, sp + k, VNG_PK);
    }
    __syncthreads();
    const int y = y0 + tid / 8, xs = x0 + (tid & 7) * 8;
    if (y >= H || xs >= W) return;
    const int cy = min(max(y, 2), H - 5), ly = cy - by;
    const bool odd_row = ((cy - 2) & 1) != 0;
    const bool green_at_2 = odd_row != (green0 != 0);
    const int blue = odd_row ? blue0 ^ 2 : blue0;
    uchar o[24];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int cx = min(max(min(xs + j, W - 1), 2), W - 3), lx = cx - bx;
        const bool green = green_at_2 != (((cx - 2) & 1) != 0);
        int c, g, oc;
        vng_pixel(sm + (ly + 2) * VNG_MW + lx + 2, VNG_MW, sp + (ly + 1) * VNG_PW + lx + 1, VNG_PW, VNG_PK, green, vng_simd_arm(cx, green_at_2, W), c, g, oc);
        o[j * 3] = (uchar)(blue ? c : oc);          // channel blueIdx gets o, blueIdx ^ 2 gets c
        o[j * 3 + 1] = (uchar)g;
        o[j * 3 + 2] = (uchar)(blue ? oc : c);
    }
    store_bytes<24>(dst.row<uchar>(f, y) + (size_t)xs * 3, min(8, W - xs) * 3, o);
}

}  // namespace

// called by b200cv_cvt_color for codes 62-65 (matrices of equal size and batch, not in place, already checked)
int demosaic_vng(const b200cvMat* src, const b200cvMat* dst, int code, cudaStream_t st)
{
    const int scn = B200CV_CN(src->type), dcn = B200CV_CN(dst->type);
    // the reference asserts an 8-bit mosaic (demosaicing.cpp:1797); it accepts dcn == 4 but writes 3-byte pixels into the 4-channel rows
    B200_REQUIRE(B200CV_DEPTH(src->type) == B200CV_8U && B200CV_DEPTH(dst->type) == B200CV_8U, "Bayer VNG needs an 8-bit mosaic and destination");
    B200_REQUIRE(scn == 1 && dcn == 3, "Bayer VNG needs a 1-channel mosaic and a 3-channel destination");
    const int W = src->cols, H = src->rows;
    if (min(W, H) < 8) return demosaic_bilinear(src, dst, 48, st);
    Img s = make_img(src), d = make_img(dst);
    if (s.frames >= 65536) return B200CV_NOT_IMPLEMENTED;
    const int c = code - 62;                                            // 0 BG, 1 GB, 2 RG, 3 GR
    const dim3 grid(div_up((unsigned)W, VNG_TW), div_up((unsigned)H, VNG_TH), (unsigned)s.frames);
    bayer_vng_kernel<<<grid, 256, 0, st>>>(s, d, W, H, c < 2 ? 0 : 2, c & 1);
    B200_LAUNCH_CHECK();
    return B200CV_OK;
}
#endif

}  // namespace b200cv
