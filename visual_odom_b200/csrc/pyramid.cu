// pyramid.cu -- K1: padded u8 Gaussian pyramid + Scharr derivative pyramid (integer, bit-exact).
//
// Replaces cv::buildOpticalFlowPyramid as run inside every cv::calcOpticalFlowPyrLK call of the
// reference's circularMatching() (reference src/feature.cpp:136-139); arithmetic restated in
// oracle/lk_ref.c (pyr_down_u8, scharr_deriv) and pinned against cv2 there.
//
//   level 0   : raw image -> REFLECT_101 padded plane                       (k_pad_level0)
//   level l+1 : 5x5 [1 4 6 4 1]^2 / 256 pyrDown of level l, written with its REFLECT_101
//               border in the same launch (border pixels recompute the reflected interior pixel)
//   derivative: Scharr of level l (reads the padded plane, so REFLECT_101 at the rim is free),
//               interior only; the border of the derivative plane stays zero (BORDER_CONSTANT).
//
// All of it is HBM/L2-bound byte work: one thread per 4 output pixels, 32-bit stores, rows are
// 64-byte aligned (pitch % 64 == 0).  No tensor cores (no contraction here).
#include "common.cuh"

static __device__ __forceinline__ uint32_t ldw(const uint8_t* p) { return __ldg(reinterpret_cast<const uint32_t*>(p)); }

// ---------------------------------------------------------------------------------------------
// raw (pitch = src_pitch) -> padded level 0.  grid.z = image index.
// src images are addressed through a pointer table (one entry per image).  With a geometry table (geo[img]: images of
// several sizes in envelope planes) the image's own size and raw pitch give the REFLECT_101 border, over the whole plane.
// SIZED (both kernels): geo is set; the other instantiation is the launch-wide-size kernel.
#define PAD_ROWS 4
template <bool SIZED>
__global__ void k_pad_level0(const uint8_t* const* __restrict__ src_tab, int src_pitch,
                             LevelGeom g, const PlaneGeom* __restrict__ geo)
{
    const int img = blockIdx.z;
    const uint8_t* __restrict__ src = src_tab[img];
    uint8_t* __restrict__ dst = g.img + (size_t)img * g.plane;
    const int wq = g.pitch >> 2;                       // 4-pixel groups per padded row
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= wq) return;
    int iw = g.w, ih = g.h;
    if (SIZED) { iw = geo[img].w[0]; ih = geo[img].h[0]; src_pitch = geo[img].pitch; }
    int sx[4];
#pragma unroll
    for (int i = 0; i < 4; i++) sx[i] = vo_reflect101(4 * q + i - VO_PAD, iw);
    // PAD_ROWS padded rows per thread: fewer, longer-lived blocks and 4 x PAD_ROWS loads in flight
    uint32_t out[PAD_ROWS];
#pragma unroll
    for (int r = 0; r < PAD_ROWS; r++) {
        const int Y = blockIdx.y * PAD_ROWS + r;           // padded row
        out[r] = 0;
        if (Y < g.hp) {
            const uint8_t* srow = src + (size_t)vo_reflect101(Y - VO_PAD, ih) * src_pitch;
#pragma unroll
            for (int i = 0; i < 4; i++) out[r] |= (uint32_t)__ldg(srow + sx[i]) << (8 * i);
        }
    }
#pragma unroll
    for (int r = 0; r < PAD_ROWS; r++) {
        const int Y = blockIdx.y * PAD_ROWS + r;
        if (Y < g.hp) *reinterpret_cast<uint32_t*>(dst + (size_t)Y * g.pitch + 4 * q) = out[r];
    }
}

// ---------------------------------------------------------------------------------------------
// One launch per level l:  (a) Scharr derivative of level l (interior),
//                          (b) if has_next: pyrDown level l -> padded level l+1.
// grid.x covers max(work_a, work_b) in units of 4 horizontally adjacent output pixels.
// With a geometry table (geo[img], level l's entries) s / d give the envelope planes and the image's own sizes give its
// border and interior: (a) writes zeros over the envelope area outside the image (the derivative border of a plane that
// held a larger image before), (b) pads level l+1 at its own size over the whole plane.
#define PYR_ROWS 1
template <bool SIZED>
__global__ void k_pyr_level(LevelGeom s, LevelGeom d, int has_next, const PlaneGeom* __restrict__ geo, int level)
{
    const int img = blockIdx.z;
    int sw = s.w, sh = s.h, dw = d.w, dh = d.h;          // the image's own sizes at levels l and l+1
    if (SIZED) {
        const PlaneGeom& g = geo[img];
        sw = g.w[level]; sh = g.h[level];
        if (has_next) { dw = g.w[level + 1]; dh = g.h[level + 1]; }
    }
    const uint8_t* __restrict__ sp = s.img + (size_t)img * s.plane + (size_t)VO_PAD * s.pitch + VO_PAD; // pixel (0,0)
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    // PYR_ROWS rows per thread (independent: the loads of all of them are in flight together, half as many blocks)
#pragma unroll
    for (int rr = 0; rr < PYR_ROWS; rr++) {
    const int row = blockIdx.y * PYR_ROWS + rr;

    // (a) derivative of level s: rows [0,h), 4 pixels per thread.  The six bytes x0-1 .. x0+4 of a row come from three
    // aligned words (x0 and the row base are multiples of 4; the padding keeps x0-4 and x0+7 inside the plane).
    if (row < s.h) {
        const int x0 = 4 * q;
        if (x0 < s.w) {
            uint32_t* __restrict__ dp = s.der + (size_t)img * s.plane + (size_t)(row + VO_PAD) * s.pitch + VO_PAD;
            uint32_t o[4] = {0u, 0u, 0u, 0u};
            if (!SIZED || (row < sh && x0 < sw)) {         // inside the image
                int t0[6], t1[6];
                {
                    int b[3][6];
#pragma unroll
                    for (int k = 0; k < 3; k++) {
                        const uint8_t* r = sp + (size_t)(row - 1 + k) * s.pitch + x0;
                        const uint32_t w0 = ldw(r - 4), w1 = ldw(r), w2 = ldw(r + 4);
                        b[k][0] = w0 >> 24; b[k][1] = w1 & 255; b[k][2] = (w1 >> 8) & 255; b[k][3] = (w1 >> 16) & 255;
                        b[k][4] = w1 >> 24; b[k][5] = w2 & 255;
                    }
#pragma unroll
                    for (int i = 0; i < 6; i++) {
                        t0[i] = (b[0][i] + b[2][i]) * 3 + b[1][i] * 10;
                        t1[i] = b[2][i] - b[0][i];
                    }
                }
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const int dx = t0[i + 2] - t0[i];
                    const int dy = (t1[i] + t1[i + 2]) * 3 + t1[i + 1] * 10;
                    o[i] = !SIZED || x0 + i < sw ? ((uint32_t)(uint16_t)(int16_t)dx) | ((uint32_t)(uint16_t)(int16_t)dy << 16) : 0u;
                }
            }
            if (x0 + 3 < s.w) {
                *reinterpret_cast<uint4*>(dp + x0) = make_uint4(o[0], o[1], o[2], o[3]);     // (PAD + x0) elements = 16-byte aligned
            } else {
#pragma unroll
                for (int i = 0; i < 4; i++)
                    if (x0 + i < s.w) dp[x0 + i] = o[i];
            }
        }
    }

    // (b) pyrDown into padded level d: padded rows [0,hp), 4 pixels per thread
    if (has_next && row < d.hp) {
        const int wq = d.pitch >> 2;
        if (q < wq) {
            uint8_t* __restrict__ dst = d.img + (size_t)img * d.plane + (size_t)row * d.pitch;
            const int dy = vo_reflect101(row - VO_PAD, dh);
            uint32_t out = 0;
            const int dx0 = 4 * q - VO_PAD;
            if (dx0 >= 0 && dx0 + 3 < dw) {
                // interior group: the 11 source bytes 2 dx0 - 2 .. 2 dx0 + 8 of a row come from four aligned words
                int acc[4] = {0, 0, 0, 0};
#pragma unroll
                for (int j = 0; j < 5; j++) {
                    const uint8_t* r = sp + (size_t)(2 * dy - 2 + j) * s.pitch + 2 * dx0;
                    const uint32_t w0 = ldw(r - 4), w1 = ldw(r), w2 = ldw(r + 4), w3 = ldw(r + 8);
                    int v[11];                                   // v[k] = source pixel 2 dx0 - 2 + k
                    v[0] = (w0 >> 16) & 255; v[1] = w0 >> 24;
                    v[2] = w1 & 255; v[3] = (w1 >> 8) & 255; v[4] = (w1 >> 16) & 255; v[5] = w1 >> 24;
                    v[6] = w2 & 255; v[7] = (w2 >> 8) & 255; v[8] = (w2 >> 16) & 255; v[9] = w2 >> 24;
                    v[10] = w3 & 255;
                    const int kj = (j == 0 || j == 4) ? 1 : ((j == 2) ? 6 : 4);
#pragma unroll
                    for (int i = 0; i < 4; i++)
                        acc[i] += kj * (v[2 * i] + v[2 * i + 4] + 4 * (v[2 * i + 1] + v[2 * i + 3]) + 6 * v[2 * i + 2]);
                }
#pragma unroll
                for (int i = 0; i < 4; i++) out |= (uint32_t)((acc[i] + 128) >> 8) << (8 * i);
            } else {
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const int dx = vo_reflect101(4 * q + i - VO_PAD, dw);
                    // source taps 2*dx-2..2*dx+2 lie inside [-2, w+1]: the REFLECT_101 border of level s
                    const uint8_t* c = sp + (size_t)(2 * dy - 2) * s.pitch + (2 * dx - 2);
                    int acc = 0;
#pragma unroll
                    for (int j = 0; j < 5; j++) {
                        const uint8_t* r = c + (size_t)j * s.pitch;
                        int h = r[0] + r[4] + 4 * (r[1] + r[3]) + 6 * r[2];
                        const int kj = (j == 0 || j == 4) ? 1 : ((j == 2) ? 6 : 4);
                        acc += kj * h;
                    }
                    out |= (uint32_t)((acc + 128) >> 8) << (8 * i);
                }
            }
            *reinterpret_cast<uint32_t*>(dst + 4 * q) = out;
        }
    }
    }   // rows of this thread
}

// ---------------------------------------------------------------------------------------------
// host launcher: builds all levels for n_img images whose raw pointers are in src_tab (device); geo: their geometry
// table entries (nullptr: every image is pg's size).  Returns the number of kernel launches issued.
int vo_launch_pyramid(const PyrGeom& pg, const uint8_t* const* src_tab_dev, int src_pitch, const PlaneGeom* geo,
                      cudaStream_t stream)
{
    int launches = 0;
    {
        const LevelGeom& g = pg.lv[0];
        dim3 block(128, 1, 1);
        dim3 grid(((g.pitch >> 2) + block.x - 1) / block.x, (g.hp + PAD_ROWS - 1) / PAD_ROWS, pg.n_img);
        if (geo) k_pad_level0<true><<<grid, block, 0, stream>>>(src_tab_dev, src_pitch, g, geo);
        else k_pad_level0<false><<<grid, block, 0, stream>>>(src_tab_dev, src_pitch, g, geo);
        launches++;
    }
    for (int l = 0; l < pg.nlevels; l++) {
        const LevelGeom& s = pg.lv[l];
        const int has_next = (l + 1 < pg.nlevels);
        const LevelGeom& d = pg.lv[has_next ? l + 1 : l];
        int qa = (s.w + 3) / 4, rows = s.h;
        if (has_next) {
            int qb = d.pitch >> 2;
            if (qb > qa) qa = qb;
            if (d.hp > rows) rows = d.hp;
        }
        dim3 block(128, 1, 1);
        dim3 grid((qa + block.x - 1) / block.x, (rows + PYR_ROWS - 1) / PYR_ROWS, pg.n_img);
        if (geo) k_pyr_level<true><<<grid, block, 0, stream>>>(s, d, has_next, geo, l);
        else k_pyr_level<false><<<grid, block, 0, stream>>>(s, d, has_next, geo, l);
        launches++;
    }
    return launches;
}
