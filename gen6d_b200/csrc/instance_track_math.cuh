// Track/detection association of the multi-instance tracker (gen6d_b200/instance_track.py) as __host__ __device__ code:
// per sequence, greedy matching of the live tracks to the re-detected instances, the update of the slot state and the
// set-up of the step's refinement chain (working poses, first-iteration dtype flags, per-iteration row lists).  track.cu
// runs it inside the re-detection step's graph, one thread per sequence of one CTA followed by a block scan that numbers
// the new tracks; its *_host entry point runs the very same per-sequence code on host memory, so the CPU tests pin it
// against a numpy restatement.  The translation unit is compiled with -fmad=false: products and sums round separately.
#pragma once
#include <math.h>
#include <stdint.h>

#include "glue_math.cuh"

namespace g6d {
namespace assoc {

constexpr int kMaxSlots = 16;      // G6D_DET_MAX_INSTANCES

struct Args {
    int S, M, F, r, num, max_misses;
    const float* det;              // [M*S,4] x, y, scale, score (instance-major: row m*S + s)
    const int* valid;              // [M*S]
    const double* init;            // [M*S,12] initial poses of the detections
    const double* cams;            // [S,20] g6d_glue_camera (K first)
    double cx, cy, cz;             // object centre
    double ref_resolution, gate;
    const double* prev;            // [M*S,12] the slots' previous poses
    int* live;                     // [M*S] in place
    long long* ids;                // [M*S] in place (-1: empty)
    int* misses;                   // [M*S] in place
    double* park;                  // [M*S,12] in place
    float* ring;                   // [M*S,num,8,2]: zeroed for spawned slots
    int* count;                    // [M*S]
    double* work;                  // [M*2S,12] out: per slot m, S real rows then S scratch rows
    uint8_t* flags0;               // [M*2S] out
    int* lists;                    // [max(F,r)*M*S] out
    int* det_slot;                 // [M*S] out
    int* spawned;                  // [M*S] out
    long long* dropped;            // [M*S] out
};

// The object centre projected with a track's previous pose and the frame's K, in fp64 and in this order:
//   p_i = ((P[i,0]*cx + P[i,1]*cy) + P[i,2]*cz) + P[i,3],  q_j = (K[j,0]*p_0 + K[j,1]*p_1) + K[j,2]*p_2,  u = q_0/q_2, v = q_1/q_2.
// Returns false when the depth q_2 is <= 0 (the track's costs are all +inf).
G6D_HD bool track_point(const double* P, const double* K, double cx, double cy, double cz, double* u, double* v) {
    double p[3], q[3];
    for (int i = 0; i < 3; ++i) p[i] = ((P[i * 4] * cx + P[i * 4 + 1] * cy) + P[i * 4 + 2] * cz) + P[i * 4 + 3];
    for (int j = 0; j < 3; ++j) q[j] = (K[j * 3] * p[0] + K[j * 3 + 1] * p[1]) + K[j * 3 + 2] * p[2];
    if (q[2] <= 0.) return false;
    *u = q[0] / q[2];
    *v = q[1] / q[2];
    return true;
}

// cost = sqrt(dx*dx + dy*dy) / (ref_resolution * scale), dx = u - x, dy = v - y (det's float32 values widened).
G6D_HD double pair_cost(double u, double v, const float* det, double ref_resolution) {
    const double dx = u - (double)det[0], dy = v - (double)det[1];
    return sqrt(dx * dx + dy * dy) / (ref_resolution * (double)det[2]);
}

G6D_HD void copy12(double* dst, const double* src) {
    for (int k = 0; k < 12; ++k) dst[k] = src[k];
}

// Everything of sequence s except the new tracks' ids; returns the number of tracks it spawns.
G6D_HD int associate_sequence(int s, const Args& a) {
    const int S = a.S, M = a.M;
    const double* K = a.cams + (long long)s * 20;
    double u[kMaxSlots], v[kMaxSlots];
    bool ok[kMaxSlots];
    for (int t = 0; t < M; ++t) {
        const long long i = (long long)t * S + s;
        ok[t] = a.live[i] && track_point(a.prev + i * 12, K, a.cx, a.cy, a.cz, &u[t], &v[t]);
    }
    // greedy matching: repeatedly the admissible pair (cost < gate) of smallest cost, ties to the lower slot, then the
    // lower detection (the scan order with a strict comparison)
    int match[kMaxSlots], det_of[kMaxSlots];
    for (int k = 0; k < M; ++k) match[k] = det_of[k] = -1;
    for (int round = 0; round < M; ++round) {
        int bt = -1, bd = -1;
        double bc = 0.;
        for (int t = 0; t < M; ++t) {
            if (!ok[t] || match[t] >= 0) continue;
            for (int d = 0; d < M; ++d) {
                const long long j = (long long)d * S + s;
                if (!a.valid[j] || det_of[d] >= 0) continue;
                const double c = pair_cost(u[t], v[t], a.det + j * 4, a.ref_resolution);
                if (c < a.gate && (bt < 0 || c < bc)) { bt = t; bd = d; bc = c; }
            }
        }
        if (bt < 0) break;
        match[bt] = bd;
        det_of[bd] = bt;
    }
    // the tracks: matched ones continue, unmatched ones miss once more and are dropped past max_misses
    int chain[kMaxSlots];
    bool is_new[kMaxSlots];
    for (int t = 0; t < M; ++t) {
        const long long i = (long long)t * S + s;
        a.dropped[i] = -1;
        is_new[t] = false;
        if (!a.live[i]) continue;
        if (match[t] >= 0) {
            a.misses[i] = 0;
        } else if (++a.misses[i] > a.max_misses) {
            a.dropped[i] = a.ids[i];
            a.live[i] = 0;
            a.ids[i] = -1;
            a.misses[i] = 0;
        }
    }
    // unmatched valid detections, in peak order, take the lowest empty slots
    int n_new = 0, t_free = 0;
    for (int d = 0; d < M; ++d) {
        const long long j = (long long)d * S + s;
        if (!a.valid[j]) { a.det_slot[j] = -1; continue; }
        if (det_of[d] >= 0) { a.det_slot[j] = det_of[d]; continue; }
        while (t_free < M && a.live[(long long)t_free * S + s]) ++t_free;
        if (t_free == M) { a.det_slot[j] = -1; continue; }
        const long long i = (long long)t_free * S + s;
        a.det_slot[j] = t_free;
        a.live[i] = 1;
        a.misses[i] = 0;
        is_new[t_free] = true;
        det_of[d] = t_free;
        copy12(a.work + ((long long)t_free * 2 * S + s) * 12, a.init + j * 12);    // the track's start: its detection's pose
        for (long long k = 0; k < (long long)a.num * 16; ++k) a.ring[i * a.num * 16 + k] = 0.f;
        a.count[i] = 0;
        ++n_new;
    }
    // every slot's start, first-iteration flag and chain length; empty slots park on detection row t of the frame
    for (int t = 0; t < M; ++t) {
        const long long i = (long long)t * S + s, real = (long long)t * 2 * S + s;
        a.spawned[i] = is_new[t];
        if (!a.live[i]) {
            copy12(a.park + i * 12, a.init + i * 12);
            a.ids[i] = -1;
        }
        double* w = a.work + real * 12;
        if (a.live[i] && !is_new[t]) copy12(w, a.prev + i * 12);
        else if (!a.live[i]) copy12(w, a.park + i * 12);
        copy12(w + (long long)S * 12, w);                                   // the scratch copy
        a.flags0[real] = a.flags0[real + S] = (uint8_t)(a.live[i] && !is_new[t]);
        chain[t] = (a.live[i] && !is_new[t]) ? a.r : a.F;
    }
    const int n_it = a.F > a.r ? a.F : a.r;
    for (int it = 0; it < n_it; ++it)
        for (int t = 0; t < M; ++t)
            a.lists[((long long)it * M + t) * S + s] = t * 2 * S + s + (it < chain[t] ? 0 : S);
    return n_new;
}

}  // namespace assoc
}  // namespace g6d
