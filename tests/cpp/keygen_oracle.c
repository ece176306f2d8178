/* halo2's permutation::keygen::Assembly restated in C, for the tests (tests/keygen_oracle.py builds it into a temporary
 * directory): the full-size comparisons of the device keygen, where the Python restatement is too slow.  Cells are flat ids
 * c 2^k + r.  For every copy (left, right), in call order, `copy` returns when both cells are in one cycle (aux), else relabels
 * the smaller cycle (sizes) with the larger one's label, walking it through mapping, and swaps mapping[left] and
 * mapping[right].  Returns 0, or -1 for a cell id >= n_cells. */
#include <stdint.h>
#include <stdlib.h>

int ko_assembly(uint32_t n_cells, const uint32_t *pairs, size_t n_pairs, uint32_t *mapping) {
    uint32_t *aux = (uint32_t *)malloc(sizeof(uint32_t) * (n_cells ? n_cells : 1));
    uint32_t *sizes = (uint32_t *)malloc(sizeof(uint32_t) * (n_cells ? n_cells : 1));
    if (!aux || !sizes) {
        free(aux);
        free(sizes);
        return -2;
    }
    for (uint32_t i = 0; i < n_cells; i++) {
        mapping[i] = i;
        aux[i] = i;
        sizes[i] = 1;
    }
    int rc = 0;
    for (size_t e = 0; e < n_pairs; e++) {
        const uint32_t left = pairs[2 * e], right = pairs[2 * e + 1];
        if (left >= n_cells || right >= n_cells) {
            rc = -1;
            break;
        }
        uint32_t left_cycle = aux[left], right_cycle = aux[right];
        if (left_cycle == right_cycle) continue;
        if (sizes[left_cycle] < sizes[right_cycle]) {
            const uint32_t t = left_cycle;
            left_cycle = right_cycle;
            right_cycle = t;
        }
        sizes[left_cycle] += sizes[right_cycle];
        uint32_t i = right_cycle;
        do {
            aux[i] = left_cycle;
            i = mapping[i];
        } while (i != right_cycle);
        const uint32_t t = mapping[left];
        mapping[left] = mapping[right];
        mapping[right] = t;
    }
    free(aux);
    free(sizes);
    return rc;
}
