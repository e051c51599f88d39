/* MPI C API of faabric_b200.  ABI-compatible with the reference's
 * include/faabric/mpi/mpi.h (same struct layouts, datatype / op ids and the
 * MPI_IN_PLACE / MPI_BOTTOM sentinels) so existing binaries keep working.
 * Extensions: 16-bit float datatypes and extra pair types for MAXLOC/MINLOC,
 * MPI_LXOR / MPI_BXOR, and buffers may be CUDA device pointers. */
#ifndef FAABRIC_B200_MPI_H
#define FAABRIC_B200_MPI_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C"
{
#endif

#define MPI_SUCCESS 0
#define MPI_ERR_OTHER 1
#define MPI_ERR_NO_MEM 2
#define MPI_ERR_OP 3
#define MPI_ERR_WIN 4
#define MPI_ERR_RANK 5
#define MPI_ERR_ARG 6
/* a synchronisation call out of place: unlock / flush of a target that is
 * not locked, a second lock, fence or free inside a passive epoch */
#define MPI_ERR_RMA_SYNC 7
#define MPI_MAX_OBJECT_NAME 128

/* passive-target lock types (MPI_Win_lock) */
#define MPI_LOCK_EXCLUSIVE 234
#define MPI_LOCK_SHARED 235

/* assert bits of MPI_Win_lock / MPI_Win_lock_all / MPI_Win_fence: NOCHECK
 * skips the lock, the others are accepted and ignored */
#define MPI_MODE_NOCHECK 1024
#define MPI_MODE_NOSTORE 2048
#define MPI_MODE_NOPUT 4096
#define MPI_MODE_NOPRECEDE 8192
#define MPI_MODE_NOSUCCEED 16384

    /* ---- opaque-ish handle structs ---- */
    struct faabric_status_public_t
    {
        int MPI_SOURCE;
        int MPI_TAG;
        int MPI_ERROR;
        int bytesSize; /* bytes actually received */
    };
    struct faabric_datatype_t
    {
        int id;
        int size;
    };
    struct faabric_communicator_t
    {
        int id;
    };
    struct faabric_message_t
    {
        int id;
    };
    struct faabric_win_t
    {
        int worldId;
        int rank;
        int size;
        void* basePtr;
        int dispUnit;
        /* window id inside the world (addition to the reference's layout) */
        int id;
        /* memory allocated by MPI_Win_allocate_shared, released by Win_free */
        void* ownedPtr;
    };
    struct faabric_op_t
    {
        int id;
    };
    struct faabric_info_t
    {
        int id;
    };
    struct faabric_request_t
    {
        int id;
    };
    struct faabric_group_t
    {
        int id;
    };

    /* ---- communicators ---- */
#define FAABRIC_COMM_WORLD 1
#define FAABRIC_COMM_NULL 2
    extern struct faabric_communicator_t faabric_comm_world;
    extern struct faabric_communicator_t faabric_comm_null;
#define MPI_COMM_WORLD &faabric_comm_world
#define MPI_COMM_NULL &faabric_comm_null

    enum
    {
        MPI_COMM_TYPE_SHARED,
    };

    /* ---- datatypes: X(ID name, numeric id, handle variable, MPI macro) ---- */
#define FAABRIC_MPI_DATATYPES(X)                                               \
    X(FAABRIC_INT8, 1, faabric_type_int8)                                      \
    X(FAABRIC_INT16, 2, faabric_type_int16)                                    \
    X(FAABRIC_INT32, 3, faabric_type_int32)                                    \
    X(FAABRIC_INT, 4, faabric_type_int)                                        \
    X(FAABRIC_INT64, 5, faabric_type_int64)                                    \
    X(FAABRIC_UINT8, 6, faabric_type_uint8)                                    \
    X(FAABRIC_UINT16, 7, faabric_type_uint16)                                  \
    X(FAABRIC_UINT32, 8, faabric_type_uint32)                                  \
    X(FAABRIC_UINT, 9, faabric_type_uint)                                      \
    X(FAABRIC_UINT64, 10, faabric_type_uint64)                                 \
    X(FAABRIC_LONG, 11, faabric_type_long)                                     \
    X(FAABRIC_LONG_LONG, 12, faabric_type_long_long)                           \
    X(FAABRIC_LONG_LONG_INT, 13, faabric_type_long_long_int)                   \
    X(FAABRIC_FLOAT, 14, faabric_type_float)                                   \
    X(FAABRIC_DOUBLE, 15, faabric_type_double)                                 \
    X(FAABRIC_DOUBLE_INT, 16, faabric_type_double_int)                         \
    X(FAABRIC_CHAR, 17, faabric_type_char)                                     \
    X(FAABRIC_C_BOOL, 18, faabric_type_c_bool)                                 \
    X(FAABRIC_BYTE, 19, faabric_type_byte)                                     \
    X(FAABRIC_DATATYPE_NULL, 20, faabric_type_null)                            \
    /* extensions */                                                           \
    X(FAABRIC_HALF, 21, faabric_type_half)                                     \
    X(FAABRIC_BFLOAT16, 22, faabric_type_bfloat16)                             \
    X(FAABRIC_FLOAT_INT, 23, faabric_type_float_int)                           \
    X(FAABRIC_2INT, 24, faabric_type_2int)                                     \
    X(FAABRIC_LONG_INT, 25, faabric_type_long_int)

#define FAABRIC_MPI_DECLARE_TYPE(name, num, var)                               \
    enum                                                                       \
    {                                                                          \
        name = num                                                             \
    };                                                                         \
    extern struct faabric_datatype_t var;
    FAABRIC_MPI_DATATYPES(FAABRIC_MPI_DECLARE_TYPE)
#undef FAABRIC_MPI_DECLARE_TYPE

#define MPI_INT8_T &faabric_type_int8
#define MPI_INT16_T &faabric_type_int16
#define MPI_INT32_T &faabric_type_int32
#define MPI_INT &faabric_type_int
#define MPI_INT64_T &faabric_type_int64
#define MPI_UINT8_T &faabric_type_uint8
#define MPI_UINT16_T &faabric_type_uint16
#define MPI_UINT32_T &faabric_type_uint32
#define MPI_UINT_T &faabric_type_uint
#define MPI_UINT64_T &faabric_type_uint64
#define MPI_LONG &faabric_type_long
#define MPI_LONG_LONG &faabric_type_long_long
#define MPI_LONG_LONG_INT &faabric_type_long_long_int
#define MPI_FLOAT &faabric_type_float
#define MPI_DOUBLE &faabric_type_double
#define MPI_DOUBLE_INT &faabric_type_double_int
#define MPI_CHAR &faabric_type_char
#define MPI_C_BOOL &faabric_type_c_bool
#define MPI_BYTE &faabric_type_byte
#define MPI_DATATYPE_NULL &faabric_type_null
#define MPI_HALF &faabric_type_half
#define MPI_BFLOAT16 &faabric_type_bfloat16
#define MPI_FLOAT_INT &faabric_type_float_int
#define MPI_2INT &faabric_type_2int
#define MPI_LONG_INT &faabric_type_long_int

    struct faabric_datatype_t* getFaabricDatatypeFromId(int datatypeId);

    /* ---- special buffer sentinels ---- */
#define FAABRIC_BOTTOM 1
#define FAABRIC_IN_PLACE 2
#define MPI_BOTTOM (void*)FAABRIC_BOTTOM
#define MPI_IN_PLACE (void*)FAABRIC_IN_PLACE

#define FAABRIC_INFO_NULL 1
#define FAABRIC_INFO_DEVICE 2
    extern struct faabric_info_t faabric_info_null;
    extern struct faabric_info_t faabric_info_device;
#define MPI_INFO_NULL &faabric_info_null
// Extension: MPI_Alloc_mem with this info allocates from the rank's symmetric
// heap in GPU memory (collective across the world)
#define MPI_INFO_FAABRIC_DEVICE &faabric_info_device

#define MPI_ANY_SOURCE -1
#define MPI_UNDEFINED -1
#define MPI_MAX_PROCESSOR_NAME 256
#define MPI_CART_MAX_DIMENSIONS 2

    /* ---- reduce operations ---- */
#define FAABRIC_MPI_OPS(X)                                                     \
    X(FAABRIC_OP_MAX, 1, faabric_op_max)                                       \
    X(FAABRIC_OP_MIN, 2, faabric_op_min)                                       \
    X(FAABRIC_OP_SUM, 3, faabric_op_sum)                                       \
    X(FAABRIC_OP_PROD, 4, faabric_op_prod)                                     \
    X(FAABRIC_OP_LAND, 5, faabric_op_land)                                     \
    X(FAABRIC_OP_LOR, 6, faabric_op_lor)                                       \
    X(FAABRIC_OP_BAND, 7, faabric_op_band)                                     \
    X(FAABRIC_OP_BOR, 8, faabric_op_bor)                                       \
    X(FAABRIC_OP_MAXLOC, 9, faabric_op_maxloc)                                 \
    X(FAABRIC_OP_MINLOC, 10, faabric_op_minloc)                                \
    X(FAABRIC_OP_NULL, 11, faabric_op_null)                                    \
    /* extensions */                                                           \
    X(FAABRIC_OP_LXOR, 12, faabric_op_lxor)                                    \
    X(FAABRIC_OP_BXOR, 13, faabric_op_bxor)                                    \
    /* one-sided accumulates only; collectives refuse them with MPI_ERR_OP */  \
    X(FAABRIC_OP_REPLACE, 14, faabric_op_replace)                              \
    X(FAABRIC_OP_NO_OP, 15, faabric_op_no_op)

#define FAABRIC_MPI_DECLARE_OP(name, num, var)                                 \
    enum                                                                       \
    {                                                                          \
        name = num                                                             \
    };                                                                         \
    extern struct faabric_op_t var;
    FAABRIC_MPI_OPS(FAABRIC_MPI_DECLARE_OP)
#undef FAABRIC_MPI_DECLARE_OP

#define MPI_MAX &faabric_op_max
#define MPI_MIN &faabric_op_min
#define MPI_SUM &faabric_op_sum
#define MPI_PROD &faabric_op_prod
#define MPI_LAND &faabric_op_land
#define MPI_LOR &faabric_op_lor
#define MPI_BAND &faabric_op_band
#define MPI_BOR &faabric_op_bor
#define MPI_MAXLOC &faabric_op_maxloc
#define MPI_MINLOC &faabric_op_minloc
#define MPI_OP_NULL &faabric_op_null
#define MPI_LXOR &faabric_op_lxor
#define MPI_BXOR &faabric_op_bxor
#define MPI_REPLACE &faabric_op_replace
#define MPI_NO_OP &faabric_op_no_op

#define MPI_STATUS_IGNORE ((MPI_Status*)(0))
#define MPI_STATUSES_IGNORE ((MPI_Status*)(0))

#define MPI_WIN_BASE 1
#define MPI_WIN_SIZE 2
#define MPI_WIN_DISP_UNIT 3
#define MPI_WIN_CREATE_FLAVOR 4
#define MPI_WIN_MODEL 5

    enum
    {
        MPI_THREAD_SINGLE,
        MPI_THREAD_FUNNELED,
        MPI_THREAD_SERIALIZED,
        MPI_THREAD_MULTIPLE
    };

    /* ---- user-facing handle types ---- */
    typedef struct faabric_op_t* MPI_Op;
    typedef struct faabric_communicator_t* MPI_Comm;
    typedef struct faabric_datatype_t* MPI_Datatype;
    typedef struct faabric_status_public_t MPI_Status;
    typedef struct faabric_message_t* MPI_Message;
    typedef struct faabric_info_t* MPI_Info;
    typedef struct faabric_request_t* MPI_Request;
    typedef struct faabric_group_t* MPI_Group;
    typedef struct faabric_win_t* MPI_Win;
    typedef ptrdiff_t MPI_Aint;
    typedef int MPI_Fint;
    typedef long MPI_Offset;

    typedef void(MPI_User_function)(void*, void*, int*, MPI_Datatype*);

    /* ---- functions ---- */
    int MPI_Init(int* argc, char*** argv);
    int MPI_Init_thread(int* argc, char*** argv, int required, int* provided);
    int MPI_Initialized(int* flag);
    int MPI_Finalized(int* flag);
    int MPI_Query_thread(int* provided);
    int MPI_Get_version(int* version, int* subversion);
    int MPI_Finalize(void);
    int MPI_Abort(MPI_Comm comm, int errorcode);
    int MPI_Get_processor_name(char* name, int* resultlen);
    double MPI_Wtime(void);

    int MPI_Comm_rank(MPI_Comm comm, int* rank);
    int MPI_Comm_size(MPI_Comm comm, int* size);
    int MPI_Comm_dup(MPI_Comm comm, MPI_Comm* newcomm);
    int MPI_Comm_free(MPI_Comm* comm);
    int MPI_Comm_split(MPI_Comm comm, int color, int key, MPI_Comm* newcomm);
    int MPI_Comm_split_type(MPI_Comm comm, int split_type, int key, MPI_Info info, MPI_Comm* newcomm);
    int MPI_Comm_create(MPI_Comm comm, MPI_Group group, MPI_Comm* newcomm);
    int MPI_Comm_create_group(MPI_Comm comm, MPI_Group group, int tag, MPI_Comm* newcomm);
    int MPI_Comm_group(MPI_Comm comm, MPI_Group* group);
    MPI_Fint MPI_Comm_c2f(MPI_Comm comm);
    MPI_Comm MPI_Comm_f2c(MPI_Fint comm);
    int MPI_Group_incl(MPI_Group group, int n, const int ranks[], MPI_Group* newgroup);
    int MPI_Group_free(MPI_Group* group);

    int MPI_Send(const void* buf, int count, MPI_Datatype datatype, int dest, int tag, MPI_Comm comm);
    int MPI_Rsend(const void* buf, int count, MPI_Datatype datatype, int dest, int tag, MPI_Comm comm);
    int MPI_Recv(void* buf, int count, MPI_Datatype datatype, int source, int tag, MPI_Comm comm, MPI_Status* status);
    int MPI_Sendrecv(const void* sendbuf, int sendcount, MPI_Datatype sendtype, int dest, int sendtag,
                     void* recvbuf, int recvcount, MPI_Datatype recvtype, int source, int recvtag,
                     MPI_Comm comm, MPI_Status* status);
    int MPI_Isend(const void* buf, int count, MPI_Datatype datatype, int dest, int tag, MPI_Comm comm, MPI_Request* request);
    int MPI_Irecv(void* buf, int count, MPI_Datatype datatype, int source, int tag, MPI_Comm comm, MPI_Request* request);
    int MPI_Wait(MPI_Request* request, MPI_Status* status);
    int MPI_Waitall(int count, MPI_Request array_of_requests[], MPI_Status* array_of_statuses);
    int MPI_Waitany(int count, MPI_Request array_of_requests[], int* index, MPI_Status* status);
    int MPI_Request_free(MPI_Request* request);
    int MPI_Probe(int source, int tag, MPI_Comm comm, MPI_Status* status);
    int MPI_Get_count(const MPI_Status* status, MPI_Datatype datatype, int* count);

    int MPI_Barrier(MPI_Comm comm);
    int MPI_Bcast(void* buffer, int count, MPI_Datatype datatype, int root, MPI_Comm comm);
    int MPI_Scatter(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
                    MPI_Datatype recvtype, int root, MPI_Comm comm);
    int MPI_Gather(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
                   MPI_Datatype recvtype, int root, MPI_Comm comm);
    int MPI_Gatherv(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf,
                    const int* recvcounts, const int* displs, MPI_Datatype recvtype, int root, MPI_Comm comm);
    int MPI_Allgather(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
                      MPI_Datatype recvtype, MPI_Comm comm);
    int MPI_Allgatherv(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf,
                       const int* recvcounts, const int* displs, MPI_Datatype recvtype, MPI_Comm comm);
    int MPI_Reduce(const void* sendbuf, void* recvbuf, int count, MPI_Datatype datatype, MPI_Op op, int root, MPI_Comm comm);
    int MPI_Reduce_scatter(const void* sendbuf, void* recvbuf, const int* recvcounts, MPI_Datatype datatype,
                           MPI_Op op, MPI_Comm comm);
    int MPI_Reduce_scatter_block(const void* sendbuf, void* recvbuf, int recvcount, MPI_Datatype datatype,
                                 MPI_Op op, MPI_Comm comm);
    int MPI_Allreduce(const void* sendbuf, void* recvbuf, int count, MPI_Datatype datatype, MPI_Op op, MPI_Comm comm);
    int MPI_Scan(const void* sendbuf, void* recvbuf, int count, MPI_Datatype datatype, MPI_Op op, MPI_Comm comm);
    int MPI_Alltoall(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
                     MPI_Datatype recvtype, MPI_Comm comm);
    int MPI_Alltoallv(const void* sendbuf, const int sendcounts[], const int sdispls[], MPI_Datatype sendtype,
                      void* recvbuf, const int recvcounts[], const int rdispls[], MPI_Datatype recvtype, MPI_Comm comm);

    int MPI_Cart_create(MPI_Comm old_comm, int ndims, const int dims[], const int periods[], int reorder, MPI_Comm* comm);
    int MPI_Cart_rank(MPI_Comm comm, int coords[], int* rank);
    int MPI_Cart_get(MPI_Comm comm, int maxdims, int dims[], int periods[], int coords[]);
    int MPI_Cart_shift(MPI_Comm comm, int direction, int disp, int* rank_source, int* rank_dest);

    int MPI_Type_size(MPI_Datatype type, int* size);
    int MPI_Type_free(MPI_Datatype* datatype);
    int MPI_Type_contiguous(int count, MPI_Datatype oldtype, MPI_Datatype* newtype);
    int MPI_Type_commit(MPI_Datatype* type);
    int MPI_Op_create(MPI_User_function* user_fn, int commute, MPI_Op* op);
    int MPI_Op_free(MPI_Op* op);

    int MPI_Alloc_mem(MPI_Aint size, MPI_Info info, void* baseptr);
    int MPI_Iallreduce(const void* sendbuf, void* recvbuf, int count, MPI_Datatype datatype, MPI_Op op, MPI_Comm comm, MPI_Request* request);
    int MPI_Ireduce_scatter_block(const void* sendbuf, void* recvbuf, int recvcount, MPI_Datatype datatype,
                                  MPI_Op op, MPI_Comm comm, MPI_Request* request);
    int MPI_Iallgather(const void* sendbuf, int sendcount, MPI_Datatype sendtype, void* recvbuf, int recvcount,
                       MPI_Datatype recvtype, MPI_Comm comm, MPI_Request* request);
    int MPI_Free_mem(void* base);
    int MPI_Win_create(void* base, MPI_Aint size, int disp_unit, MPI_Info info, MPI_Comm comm, MPI_Win* win);
    int MPI_Win_allocate_shared(MPI_Aint size, int disp_unit, MPI_Info info, MPI_Comm comm, void* baseptr, MPI_Win* win);
    int MPI_Win_shared_query(MPI_Win win, int rank, MPI_Aint* size, int* disp_unit, void* baseptr);
    int MPI_Win_fence(int assert, MPI_Win win);
    int MPI_Win_free(MPI_Win* win);
    int MPI_Win_get_attr(MPI_Win win, int win_keyval, void* attribute_val, int* flag);
    int MPI_Get(void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
                MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Win win);
    int MPI_Put(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
                MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Win win);
    /* One-sided atomics: every target element is updated atomically.  Fetched
     * values are defined after the closing MPI_Win_fence. */
    int MPI_Accumulate(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
                       MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Op op, MPI_Win win);
    int MPI_Get_accumulate(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype,
                           void* result_addr, int result_count, MPI_Datatype result_datatype, int target_rank,
                           MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Op op,
                           MPI_Win win);
    int MPI_Fetch_and_op(const void* origin_addr, void* result_addr, MPI_Datatype datatype, int target_rank,
                         MPI_Aint target_disp, MPI_Op op, MPI_Win win);
    int MPI_Compare_and_swap(const void* origin_addr, const void* compare_addr, void* result_addr,
                             MPI_Datatype datatype, int target_rank, MPI_Aint target_disp, MPI_Win win);
    /* Passive-target synchronisation.  Inside a lock epoch, operations are
     * complete at origin and target (fetched values defined) after
     * MPI_Win_flush* or MPI_Win_unlock* of their target; no fence. */
    int MPI_Win_lock(int lock_type, int rank, int assert, MPI_Win win);
    int MPI_Win_unlock(int rank, MPI_Win win);
    int MPI_Win_lock_all(int assert, MPI_Win win);
    int MPI_Win_unlock_all(MPI_Win win);
    int MPI_Win_flush(int rank, MPI_Win win);
    int MPI_Win_flush_all(MPI_Win win);
    int MPI_Win_flush_local(int rank, MPI_Win win);
    int MPI_Win_flush_local_all(MPI_Win win);
    int MPI_Win_sync(MPI_Win win);
    /* Request-based operations, inside a passive epoch that covers the
     * target.  After MPI_Wait* on the request the origin buffer may be reused
     * (put, accumulate) or holds the data (get, get-accumulate).
     * MPI_Win_flush* and MPI_Win_unlock* complete them too. */
    int MPI_Rput(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
                 MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Win win,
                 MPI_Request* request);
    int MPI_Rget(void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
                 MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Win win,
                 MPI_Request* request);
    int MPI_Raccumulate(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype, int target_rank,
                        MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Op op,
                        MPI_Win win, MPI_Request* request);
    int MPI_Rget_accumulate(const void* origin_addr, int origin_count, MPI_Datatype origin_datatype,
                            void* result_addr, int result_count, MPI_Datatype result_datatype, int target_rank,
                            MPI_Aint target_disp, int target_count, MPI_Datatype target_datatype, MPI_Op op,
                            MPI_Win win, MPI_Request* request);

#ifdef __cplusplus
}
#endif

#endif
