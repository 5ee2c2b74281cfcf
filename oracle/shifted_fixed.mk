# oracle/shifted_fixed.mk -- the checker of shifted_lopbicg (shifted_switching_solver.h:11).  TEST INFRASTRUCTURE, never the product.
# It includes oracle/Makefile for its variables and adds:
#
#   make -f shifted_fixed.mk fixed-oracle   liboracle_fixed.so : the C restatement (shifted_fixed_oracle.c), strict IEEE
#
# The reference's own shifted_lopbicg needs no recipe of its own: oracle/Makefile already links the whole of
# shifted_switching_solver.c into _ref/libref_strict.so.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := fixed-oracle
.PHONY: fixed-oracle

fixed-oracle: $(HERE)liboracle_fixed.so
$(HERE)liboracle_fixed.so: $(HERE)shifted_fixed_oracle.c $(HERE)bicg_oracle.c
	$(CC) $(STRICT) -std=c11 -fPIC -shared -Wall -Wextra -o $@ $< -lm
