/*
 * kxpu_oracle.h -- the oracle functions that one file of libkxpu_oracle.so calls in another.  The defining file and
 * every calling file include it, so the compiler checks each call against the definition.
 *
 * TEST INFRASTRUCTURE ONLY, like kxpu_oracle.c.
 */
#ifndef KXPU_ORACLE_H
#define KXPU_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#include "../include/kxpu.h"

/* kxpu_oracle.c: the yaml.v3 base-60 predicate, so every oracle's documents quote the same bdf strings */
int kxo_is_base60(const uint8_t *s, size_t len);

/* kxpu_xpu_oracle.c: the CDI kind domain and the any-vendor grouping */
int kxo_kind_ok(const char *kind);
int32_t kxo_classify_rules(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs, size_t n,
                           kxpu_classify_out *out, uint8_t *dev_rule);

/* kxpu_mdev_oracle.c: the vGPU grouping */
int32_t kxo_mdev_classify(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_mdevrec *recs, size_t n,
                          kxpu_classify_out *out, uint8_t *dev_rule);

/* kxpu_topo_oracle.c: the any-vendor grouping with per-group NUMA masks */
int32_t kxo_classify_topo(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs, size_t n,
                          kxpu_classify_out *out, uint8_t *dev_rule, uint64_t *group_numa);

#endif
