# oracle/shifted_lop.mk -- the checker of the LOP family of shifted_solver.h.  TEST INFRASTRUCTURE, never the product.
# It includes oracle/Makefile for its variables and object rules, and adds:
#
#   make -f shifted_lop.mk lop-oracle   liboracle_lop.so : the C restatement (shifted_lop_oracle.c), strict IEEE
#   make -f shifted_lop.mk lop-ref      _ref/* (only when $(REF)/src exists; only binaries land in oracle/_ref/):
#     _ref/libref_lop_strict.so       shifted_solver.c patched like shifted_switching_solver.c (oracle/Makefile) +
#                                     -DDISPLAY_RESIDUAL, -O2 -ffp-contract=off: bit-for-bit partner of liboracle_lop.so
#     _ref/ref_test_shifted_stock     the reference's test_shifted.c UNMODIFIED with its own sources on the mini-MPI
#     _ref/ref_test_shifted_b200      the same test_shifted.c, UNCHANGED, linked against libbicgstab_b200.so
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := lop-oracle
.PHONY: lop-oracle lop-ref

lop-oracle: $(HERE)liboracle_lop.so
$(HERE)liboracle_lop.so: $(HERE)shifted_lop_oracle.c $(HERE)bicg_oracle.c
	$(CC) $(STRICT) -std=c11 -fPIC -shared -Wall -Wextra -o $@ $< -lm

ifneq ($(wildcard $(SRC)/shifted_solver.c),)
lop-ref: $(OUT)/libref_lop_strict.so $(OUT)/ref_test_shifted_stock $(OUT)/ref_test_shifted_b200
else
lop-ref:
	@echo "oracle: $(SRC)/shifted_solver.c not present -- using prebuilt oracle/_ref if any"
endif

$(OUT)/shifted_solver_strict.o: $(SRC)/shifted_solver.c $(HERE)ref_shim.h | $(OUT)
	$(SEDPATCH) $(SRC)/shifted_solver.c | $(CC) $(STRICT) $(WARN) -fPIC $(INC) -DDISPLAY_RESIDUAL -include $(HERE)ref_shim.h -x c -c - -o $@

$(OUT)/libref_lop_strict.so: $(OUT)/shifted_solver_strict.o $(OUT)/matrix_strict.o $(OUT)/vector_strict.o $(OUT)/mmio_strict.o $(SUPPORT)
	$(CC) -shared -Wl,-Bsymbolic -o $@ $^ -lm

$(OUT)/ref_test_shifted_stock: $(SRC)/test_shifted.c $(SRC)/shifted_solver.c $(SRC)/matrix.c $(SRC)/vector.c $(SRC)/mmio.c $(OUT)/mini_mpi.o
	$(CC) $(FAST) $(WARN) $(INC) -o $@ $^ -lm
$(OUT)/ref_test_shifted_b200: $(SRC)/test_shifted.c $(B200LIB)/libbicgstab_b200.so | $(OUT)
	$(CC) -O2 $(WARN) -I$(abspath $(HERE)../include/compat) -I$(SRC) $(SRC)/test_shifted.c -L$(B200LIB) -lbicgstab_b200 \
	      -Wl,-rpath,'$$ORIGIN/../../mpi-bicgstab_b200' -o $@ -lm
