// Track/detection association of the multi-instance trackers (gen6d_b200/instance_track.py) as __host__ __device__ code:
// per (sequence, object) pair, greedy matching of the pair's live tracks to its re-detected instances, the update of the
// slot state and the set-up of the step's refinement chain (working poses, first-iteration dtype flags, per-iteration row
// lists).  track.cu runs it inside the re-detection step's graph, one thread per pair of one CTA followed by a block scan
// that numbers the new tracks; its *_host entry points run the very same per-pair code on host memory, so the CPU tests
// pin it against a numpy restatement.  The translation unit is compiled with -fmad=false: products and sums round
// separately.
//
// A step in which only some sequences re-detect (g6d_instances_associate_sequences) gives each sequence its row j in a
// detection batch of D rows per slot group (det_index[s], -1: the sequence does not detect): the detecting pairs run the
// association on detection rows g*D + j, the others only set up their refinement, as a refine-only step does.
//
// A verifying step (g6d_instances_verify_update, row f21) feeds the same miss rule (track_seen): a live slot judged lost
// is a track not seen, one judged found a track matched.
//
// Layout: K objects with M instance slots each over S sequences; slot group g = m*K + o is instance slot m of object o,
// and row g*S + s is that slot on sequence s.  A single object (g6d_instances_associate) is K = 1, where g = m and every
// row index, work row and id is the one of the single-object layout.
#pragma once
#include <math.h>
#include <stdint.h>

#include "glue_math.cuh"

namespace g6d {
namespace assoc {

constexpr int kMaxSlots = 16;      // G6D_DET_MAX_INSTANCES

struct Args {
    int S, K, M, F, r, num, max_misses;
    const float* det;              // [M*K*S,4] x, y, scale, score (row g*S + s, g = m*K + o)
    const int* valid;              // [M*K*S]
    const double* init;            // [M*K*S,12] initial poses of the detections
    const double* cams;            // [S,20] g6d_glue_camera (K first)
    const double* centers;         // [K,3] the objects' centres, or null: center1 for the single object
    double center1[3];
    double ref_resolution, gate;
    const double* prev;            // [M*K*S,12] the slots' previous poses
    int* live;                     // [M*K*S] in place
    long long* ids;                // [M*K*S] in place (-1: empty)
    int* misses;                   // [M*K*S] in place
    double* park;                  // [M*K*S,12] in place
    float* ring;                   // [M*K*S,num,8,2]: zeroed for spawned slots
    int* count;                    // [M*K*S]
    double* work;                  // [M*K*2S,12] out: per slot group g, S real rows g*2S + s then S scratch rows
    uint8_t* flags0;               // [M*K*2S] out
    int* lists;                    // [max(F,r)*M*K*S] out: entry (it*M*K + g)*S + s
    int* det_slot;                 // [M*K*S] out
    int* spawned;                  // [M*K*S] out
    long long* dropped;            // [M*K*S] out
    const int* det_index;          // [S] each sequence's detection row j < D, -1: no detection; null: every s detects at s, D = S
    int D;                         // detection rows per slot group (det, valid, init are [M*K*D,...], row g*D + j)
};

G6D_HD int det_rows(const Args& a) { return a.det_index ? a.D : a.S; }

// The entry of lists for slot t (slot group g = t*K + o) at iteration it: iterations it < r list every row of the
// M*K*S (entry (it*M*K + g)*S + s); iterations r <= it < F follow with the M*K*D rows of the detecting sequences only
// (entry r*M*K*S + ((it - r)*M*K + g)*D + j).  With det_index null (D = S, j = s) both are (it*M*K + g)*S + s.
G6D_HD long long list_entry(const Args& a, int it, int g, int s, int j) {
    const long long G = (long long)a.M * a.K;
    if (it < a.r) return ((long long)it * G + g) * a.S + s;
    return (long long)a.r * G * a.S + ((long long)(it - a.r) * G + g) * det_rows(a) + j;
}

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

// Live slot i after a look at its frame: seen (matched to a detection, or judged found by verification) restarts its
// misses; not seen takes a miss and is dropped past max_misses (live 0, ids -1, misses 0, its id written to dropped[i]).
G6D_HD void track_seen(long long i, bool seen, int max_misses, int* live, long long* ids, int* misses, long long* dropped) {
    if (seen) {
        misses[i] = 0;
    } else if (++misses[i] > max_misses) {
        dropped[i] = ids[i];
        live[i] = 0;
        ids[i] = -1;
        misses[i] = 0;
    }
}

// The verification update of row i (g6d_instances_verify_update): dropped[i] = -1, then a live slot of a verified row is
// seen unless judged lost.  Empty slots and unverified rows keep their state.
G6D_HD void verify_update(long long i, const int* lost, const int* verified, int max_misses, int* live, long long* ids, int* misses,
                          long long* dropped) {
    dropped[i] = -1;
    if (verified[i] && live[i]) track_seen(i, !lost[i], max_misses, live, ids, misses, dropped);
}

// Everything of sequence s and object o except the new tracks' ids; returns the number of tracks it spawns.  The pair's
// slot t is row base + t*stride (base = o*S + s, stride = K*S: slot group g = t*K + o) and matches only its object's
// detection rows, with its object's centre.
G6D_HD int setup_refinement(int s, int o, const Args& a);

G6D_HD int associate_sequence(int s, int o, const Args& a) {
    const int S = a.S, M = a.M;
    const int jd = a.det_index ? a.det_index[s] : s;                   // the sequence's row in the detection batch
    if (jd < 0) return setup_refinement(s, o, a);
    const long long base = (long long)o * S + s, stride = (long long)a.K * S;
    const long long dbase = (long long)o * det_rows(a) + jd, dstride = (long long)a.K * det_rows(a);
    const double* K = a.cams + (long long)s * 20;
    const double* c = a.centers ? a.centers + (long long)o * 3 : a.center1;
    const double cx = c[0], cy = c[1], cz = c[2];
    double u[kMaxSlots], v[kMaxSlots];
    bool ok[kMaxSlots];
    for (int t = 0; t < M; ++t) {
        const long long i = base + t * stride;
        ok[t] = a.live[i] && track_point(a.prev + i * 12, K, cx, cy, cz, &u[t], &v[t]);
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
                const long long j = dbase + d * dstride;
                if (!a.valid[j] || det_of[d] >= 0) continue;
                const double cost = pair_cost(u[t], v[t], a.det + j * 4, a.ref_resolution);
                if (cost < a.gate && (bt < 0 || cost < bc)) { bt = t; bd = d; bc = cost; }
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
        const long long i = base + t * stride;
        a.dropped[i] = -1;
        is_new[t] = false;
        if (!a.live[i]) continue;
        track_seen(i, match[t] >= 0, a.max_misses, a.live, a.ids, a.misses, a.dropped);
    }
    // work row of slot t: its group's S real rows, then S scratch rows
    auto real_row = [&](int t) { return (long long)(t * a.K + o) * 2 * S + s; };
    // unmatched valid detections, in peak order, take the lowest empty slots
    int n_new = 0, t_free = 0;
    for (int d = 0; d < M; ++d) {
        const long long j = dbase + d * dstride, q = base + d * stride;     // detection d's batch row and its det_slot row
        if (!a.valid[j]) { a.det_slot[q] = -1; continue; }
        if (det_of[d] >= 0) { a.det_slot[q] = det_of[d]; continue; }
        while (t_free < M && a.live[base + t_free * stride]) ++t_free;
        if (t_free == M) { a.det_slot[q] = -1; continue; }
        const long long i = base + t_free * stride;
        a.det_slot[q] = t_free;
        a.live[i] = 1;
        a.misses[i] = 0;
        is_new[t_free] = true;
        det_of[d] = t_free;
        copy12(a.work + real_row(t_free) * 12, a.init + j * 12);           // the track's start: its detection's pose
        for (long long k = 0; k < (long long)a.num * 16; ++k) a.ring[i * a.num * 16 + k] = 0.f;
        a.count[i] = 0;
        ++n_new;
    }
    // every slot's start, first-iteration flag and chain length; empty slots park on detection row t of the frame
    for (int t = 0; t < M; ++t) {
        const long long i = base + t * stride, real = real_row(t);
        a.spawned[i] = is_new[t];
        if (!a.live[i]) {
            copy12(a.park + i * 12, a.init + (dbase + t * dstride) * 12);
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
            a.lists[list_entry(a, it, t * a.K + o, s, jd)] = (int)real_row(t) + (it < chain[t] ? 0 : S);
    return n_new;
}

// A pair that does not detect this step: the set-up of a refine-only step (work row = live ? prev : park and its scratch
// copy, flags0 = live, chain r, listed in iterations it < r), spawned 0, dropped and det_slot -1; the slot state is not
// touched.
G6D_HD int setup_refinement(int s, int o, const Args& a) {
    const int S = a.S;
    const long long base = (long long)o * S + s, stride = (long long)a.K * S;
    for (int t = 0; t < a.M; ++t) {
        const long long i = base + t * stride, real = (long long)(t * a.K + o) * 2 * S + s;
        double* w = a.work + real * 12;
        copy12(w, a.live[i] ? a.prev + i * 12 : a.park + i * 12);
        copy12(w + (long long)S * 12, w);
        a.flags0[real] = a.flags0[real + S] = (uint8_t)a.live[i];
        a.spawned[i] = 0;
        a.dropped[i] = -1;
        a.det_slot[i] = -1;
        for (int it = 0; it < a.r; ++it) a.lists[list_entry(a, it, t * a.K + o, s, -1)] = (int)real;
    }
    return 0;
}

// Detection row j < D that no sequence uses (padding of the detection batch): in iterations r <= it < F its M*K list
// entries point at the scratch rows of the rank-th non-detecting sequence, rank = j's rank among the unused rows.  Those
// rows are free (a non-detecting chain ends at r) and there are enough of them (D - #detecting <= S - #detecting), so a
// padding entry never refines a real row nor shares a row with another entry.
G6D_HD void pad_lists(int j, const Args& a) {
    int below = 0;
    for (int s = 0; s < a.S; ++s) {
        if (a.det_index[s] == j) return;
        below += a.det_index[s] >= 0 && a.det_index[s] < j;
    }
    int rank = j - below, s = 0;
    for (; s < a.S; ++s)
        if (a.det_index[s] < 0 && rank-- == 0) break;
    const int n_it = a.F > a.r ? a.F : a.r;
    for (int it = a.r; it < n_it; ++it)
        for (int g = 0; g < a.M * a.K; ++g) a.lists[list_entry(a, it, g, s, j)] = g * 2 * a.S + a.S + s;
}

}  // namespace assoc
}  // namespace g6d
