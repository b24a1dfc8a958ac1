# Compiles the reference's two marching-cubes tables (edge_table_ and triangle_table_ of
# libintrinsic3d/src/mesh/marching_cubes.cpp) into oracle/_ref/libmc_ref_tables.so, read from the reference tree at build time.
# tests/test_mesh.py pins the generated tables of intrinsic3d_b200/csrc/gen_mc_tables.py against it.  The extracted source and the
# library stay under oracle/_ref/, which git ignores: the tables never enter the repository.
#   make -C oracle -f mc_ref.mk I3D_REFERENCE=<reference tree>
I3D_REFERENCE ?= /root/reference
CXX := /usr/bin/g++
SRC := $(I3D_REFERENCE)/libintrinsic3d/src/mesh/marching_cubes.cpp
OUT := _ref

all: $(OUT)/libmc_ref_tables.so

# each table: the initialiser after "<name> =" up to the first line that closes it with "};"
$(OUT)/mc_ref_tables.cpp: $(SRC) mc_ref.mk
	mkdir -p $(OUT)
	{ echo 'extern "C" const int i3d_ref_edge_table[256] ='; \
	  awk '/edge_table_\[256\] *=/ { f = 1; sub(/.*=/, "") } f { print } f && /};/ { exit }' $(SRC); \
	  echo 'extern "C" const int i3d_ref_triangle_table[256][16] ='; \
	  awk '/triangle_table_\[256\]\[16\] *=/ { f = 1; sub(/.*=/, "") } f { print } f && /};/ { exit }' $(SRC); } > $@.tmp
	mv $@.tmp $@

$(OUT)/libmc_ref_tables.so: $(OUT)/mc_ref_tables.cpp
	$(CXX) -O0 -fPIC -shared -o $@ $<

clean:
	rm -f $(OUT)/mc_ref_tables.cpp $(OUT)/libmc_ref_tables.so
