// OpenCV 4.13 candidate hierarchy (SURVEY A.5, DESIGN.md finding 2) for host and device: which selected candidates
// identification reaches.  k_rejected uses it to gather detectMarkers' rejectedImgPoints, and tests/hostsim/rejected_hostsim.cpp to
// check the markers and the rejected list against cv2 on the CPU.  k_finish states the same loop inline: called through these
// functions it compiled to another instruction schedule (same registers, stack and spills), and its SASS is kept as it is.
#pragma once
#include "common.cuh"
#include "quad_group.cuh"

namespace fid {

// Candidates are in descending-perimeter order; the parent of i is the nearest larger candidate whose quad contains all four
// corners of i, -1 for none.  qi = the quad of i, quad(j) = the quad of selected candidate j.
template <class QuadOf>
FID_HD int tree_parent(const QuadF& qi, int i, const QuadOf& quad) {
    int parent = -1;
    for (int j = i - 1; j >= 0; j--)
        if (quad_inside_quad(qi, quad(j))) {
            parent = j;
            break;
        }
    return parent;
}

// The level loop over the ns candidates with parents `parent` (tree_parent); depth[] and was[] start at 0.  decoded(v) = candidate
// v was identified.  Afterwards was[v] bit 1 says that v's level was reached: the candidate is a marker when it also decoded, and
// rejected otherwise.
template <class Decoded>
FID_HD void tree_levels(int ns, const short* parent, short* depth, unsigned char* was, const Decoded& decoded) {
    // depth: leaves 0, a parent one more than its deepest child (children have larger indices)
    int max_depth = 0;
    for (int i = ns - 1; i >= 0; i--) {
        const int p = parent[i];
        if (p >= 0 && depth[p] < depth[i] + 1) depth[p] = (short)(depth[i] + 1);
        max_depth = depth[i] > max_depth ? depth[i] : max_depth;
    }
    // identification runs level by level, innermost first, `while (counter < ncandidates)`: an identified candidate
    // counts all its not yet visited ancestors, every candidate of a level counts itself once more -- so the loop can end
    // before the outer levels are reached (a marker that encloses an identified marker is then never looked at), but a
    // level that is reached is identified completely.  was[i] bit 1 = level reached ("processed").
    int counter = 0;
    for (int d = 0; d <= max_depth && counter < ns; d++) {
        for (int v = 0; v < ns; v++)
            if (depth[v] == d) was[v] |= 3;
        for (int v = 0; v < ns; v++) {
            if (depth[v] != d) continue;
            if (decoded(v))
                for (int p = parent[v]; p != -1; p = parent[p])
                    if (!(was[p] & 1)) {
                        was[p] |= 1;
                        counter++;
                    }
            counter++;
        }
    }
}

}  // namespace fid
